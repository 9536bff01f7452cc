// The scene-flow figure of the reference's visualize_scene_flow (utils/visualization_tools.py:729-821).  Per sampled
// frame the reference runs seven boolean indexes on the flow class, the camera mask of get_valid_lidar_mask
// (datasets/waymo.py:638-668: per camera an inverse() that syncs and a matmul projection) with seven more boolean
// indexes, and two scene_flow_to_rgb calls with their masked assignments.  Here:
//
// emer_flow_vis_select: one launch per frame.  Per point: the class filter, the camera test against num_cams 4x4
//   lidar2img matrices, and, for a kept point, its coordinates, timestamp and label colour appended in point order
//   behind the running count (the chained tile scan of ordered_scan.cuh).  The frame's labelled and kept counts are
//   added to its row of a counts array with integer atomics.
// emer_flow_vis_color: one thread per row: the dynamic-density gate (x *= 0 where density < threshold) and the colour
//   of flow_color.cuh; or, for scene_flow_to_rgb's quantile, the unscaled radius alone.
//
// Arithmetic is the reference's fp32 with one rounding per torch op.
#include "common.cuh"
#include "flow_color.cuh"
#include "ordered_scan.cuh"

namespace emer {

constexpr int FV_THREADS = 256;
constexpr int FV_ROWS_PER_THREAD = EMER_FLOW_VIS_TILE / FV_THREADS;
constexpr int FV_MAX_TILES = EMER_FLOW_VIS_MAX_ROWS / EMER_FLOW_VIS_TILE;
static_assert(FV_ROWS_PER_THREAD * FV_THREADS == EMER_FLOW_VIS_TILE, "tile rows");
static_assert(8 + 8 * (size_t)FV_MAX_TILES <= EMER_FLOW_VIS_WORKSPACE_BYTES, "select workspace");

struct SelectParams {
    const float *origins, *viewdirs, *ranges, *times, *flows;
    int64_t ld_origins, ld_viewdirs, ld_ranges, ld_times, ld_flows;
    const int64_t* classes;
    int64_t ld_classes;
    const float* lidar2img;                        // [cams, 4, 4]
    int cams;
    float width, height;
    int64_t n, tiles;
    float *points, *out_times, *rows9;
    long long *count, *frame_counts;
    unsigned int* ticket;
    unsigned long long* flags;
};

// The reference's lidar point origin + range * viewdir (two roundings).
__device__ __forceinline__ void lidar_point(const SelectParams& p, int64_t r, float q[3]) {
    const float t = __ldg(p.ranges + r * p.ld_ranges);
#pragma unroll
    for (int a = 0; a < 3; ++a)
        q[a] = __fadd_rn(__ldg(p.origins + r * p.ld_origins + a), __fmul_rn(t, __ldg(p.viewdirs + r * p.ld_viewdirs + a)));
}

// get_valid_lidar_mask for one point: (M[:3, :3] @ q + M[:3, 3]) per camera, the fp32 product a k-ordered fma chain
// and the translation added separately; u, v = xy / (depth + 1e-6); kept when 0 <= u < W, 0 <= v < H and depth > 0 in
// any camera.
__device__ __forceinline__ bool in_view(const float* m, int cams, float w, float h, const float q[3]) {
    bool seen = false;
    for (int c = 0; c < cams; ++c) {
        const float* M = m + 16 * c;
        float pr[3];
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            float acc = 0.0f;
#pragma unroll
            for (int k = 0; k < 3; ++k) acc = fmaf(M[4 * r + k], q[k], acc);
            pr[r] = __fadd_rn(acc, M[4 * r + 3]);
        }
        const float den = __fadd_rn(pr[2], 1e-6f);
        const float u = __fdiv_rn(pr[0], den), v = __fdiv_rn(pr[1], den);
        seen |= u >= 0.0f && u < w && v >= 0.0f && v < h && pr[2] > 0.0f;
    }
    return seen;
}

__global__ void __launch_bounds__(FV_THREADS) flow_vis_select_kernel(const SelectParams p) {
    __shared__ long long sh[FV_THREADS / 32];
    __shared__ long long round_base[FV_ROWS_PER_THREAD + 1];
    __shared__ long long tile_base;
    __shared__ int64_t tile_s;
    __shared__ float m[16 * EMER_FLOW_VIS_MAX_CAMS];
    for (int i = threadIdx.x; i < 16 * p.cams; i += FV_THREADS) m[i] = __ldg(p.lidar2img + i);
    if (threadIdx.x == 0) tile_s = take_tile(p.ticket);
    __syncthreads();
    const int64_t tile = tile_s;
    const int64_t r0 = tile * EMER_FLOW_VIS_TILE;
    // rows r0 + i * FV_THREADS + threadIdx.x: coalesced reads, and (round, thread) order is row order
    unsigned keep = 0;
    long long labelled = 0;
#pragma unroll
    for (int i = 0; i < FV_ROWS_PER_THREAD; ++i) {
        const int64_t r = r0 + (int64_t)i * FV_THREADS + threadIdx.x;
        if (r >= p.n || __ldg(p.classes + r * p.ld_classes) == -1) continue;
        ++labelled;
        float q[3];
        lidar_point(p, r, q);
        if (in_view(m, p.cams, p.width, p.height, q)) keep |= 1u << i;
    }
    int mine[FV_ROWS_PER_THREAD];                     // offset of the row in its round (< FV_THREADS)
    long long acc = 0, labelled_all;
    block_exclusive_scan<FV_THREADS>(labelled, sh, &labelled_all);
#pragma unroll
    for (int i = 0; i < FV_ROWS_PER_THREAD; ++i) {
        long long total;
        mine[i] = (int)block_exclusive_scan<FV_THREADS>((keep >> i) & 1u, sh, &total);
        if (threadIdx.x == 0) round_base[i] = acc;
        acc += total;
    }
    if (threadIdx.x == 0) {
        tile_base = chain_tile(tile, p.tiles, acc, p.count, p.ticket, p.flags);
        atomicAdd((unsigned long long*)p.frame_counts, (unsigned long long)labelled_all);
        atomicAdd((unsigned long long*)p.frame_counts + 1, (unsigned long long)acc);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < FV_ROWS_PER_THREAD; ++i) {
        if (!((keep >> i) & 1u)) continue;
        const int64_t r = r0 + (int64_t)i * FV_THREADS + threadIdx.x;
        const long long o = tile_base + round_base[i] + mine[i];
        float q[3], rgb[3];
        lidar_point(p, r, q);
        const float* f = p.flows + r * p.ld_flows;
        flow_rgb(__ldg(f), __ldg(f + 1), FLOW_SCALE_HOST, 0.5f, true, rgb);     // flow_max_radius=2.0, "bright"
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            p.points[3 * o + a] = q[a];
            p.rows9[9 * o + a] = q[a];
            p.rows9[9 * o + 6 + a] = rgb[a];
        }
        p.out_times[o] = __ldg(p.times + r * p.ld_times);
    }
}

struct ColorParams {
    const float* flow;
    int64_t ld_flow;
    const float* density;
    float threshold;
    int64_t n;
    int scale_mode;
    float scale;
    const float* device_radius;
    bool bright;
    float* colors;
    int64_t ld_colors;
    float* radius;
};

__global__ void __launch_bounds__(FV_THREADS) flow_vis_color_kernel(const ColorParams p) {
    const int64_t r = (int64_t)blockIdx.x * FV_THREADS + threadIdx.x;
    if (r >= p.n) return;
    float x = __ldg(p.flow + r * p.ld_flow), y = __ldg(p.flow + r * p.ld_flow + 1);
    if (p.density && __ldg(p.density + r) < p.threshold) {     // pred[dynamic_density < thr] *= 0: NaN is not gated
        x = __fmul_rn(x, 0.0f);
        y = __fmul_rn(y, 0.0f);
    }
    if (!p.colors) {
        float angle;
        flow_polar(x, y, p.radius[r], angle);
        return;
    }
    const float scale = p.scale_mode == FLOW_SCALE_DEVICE ? __ldg(p.device_radius) : p.scale;
    float rgb[3];
    flow_rgb(x, y, p.scale_mode, scale, p.bright, rgb);
    float* out = p.colors + r * p.ld_colors;
    out[0] = rgb[0];
    out[1] = rgb[1];
    out[2] = rgb[2];
}

}  // namespace emer

using namespace emer;

extern "C" int emer_flow_vis_select(const float* origins, int64_t ld_origins, const float* viewdirs,
                                    int64_t ld_viewdirs, const float* ranges, int64_t ld_ranges, const float* times,
                                    int64_t ld_times, const float* flows, int64_t ld_flows, const int64_t* classes,
                                    int64_t ld_classes, int64_t n, const float* lidar2img, int num_cams, float width,
                                    float height, float* points, float* out_times, float* rows9, int64_t* count,
                                    int64_t* frame_counts, void* workspace, void* stream) {
    const char* what = "emer_flow_vis_select";
    EMER_REQUIRE(n >= 0 && n <= EMER_FLOW_VIS_MAX_ROWS, "%s: %lld points (at most %d)", what, (long long)n,
                 EMER_FLOW_VIS_MAX_ROWS);
    EMER_REQUIRE(num_cams >= 1 && num_cams <= EMER_FLOW_VIS_MAX_CAMS, "%s: %d cameras (1..%d)", what, num_cams,
                 EMER_FLOW_VIS_MAX_CAMS);
    EMER_REQUIRE(count && frame_counts && workspace, "%s: NULL pointer", what);
    if (n == 0) return 0;
    EMER_REQUIRE(origins && viewdirs && ranges && times && flows && classes && lidar2img && points && out_times && rows9,
                 "%s: NULL pointer", what);
    EMER_REQUIRE(ld_origins >= 3 && ld_viewdirs >= 3 && ld_ranges >= 1 && ld_times >= 1 && ld_flows >= 3 &&
                     ld_classes >= 1,
                 "%s: row strides", what);
    SelectParams p{};
    p.origins = origins; p.viewdirs = viewdirs; p.ranges = ranges; p.times = times; p.flows = flows;
    p.ld_origins = ld_origins; p.ld_viewdirs = ld_viewdirs; p.ld_ranges = ld_ranges; p.ld_times = ld_times;
    p.ld_flows = ld_flows;
    p.classes = classes; p.ld_classes = ld_classes;
    p.lidar2img = lidar2img; p.cams = num_cams; p.width = width; p.height = height;
    p.n = n; p.tiles = ceil_div(n, EMER_FLOW_VIS_TILE);
    p.points = points; p.out_times = out_times; p.rows9 = rows9;
    p.count = (long long*)count; p.frame_counts = (long long*)frame_counts;
    p.ticket = (unsigned int*)workspace;
    p.flags = (unsigned long long*)((unsigned char*)workspace + 8);
    flow_vis_select_kernel<<<(int)p.tiles, FV_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch(what);
}

extern "C" int emer_flow_vis_color(const float* flow, int64_t ld_flow, const float* density, float threshold,
                                   int64_t n, int scale_mode, float radius_scale, const float* device_radius,
                                   int bright, float* colors, int64_t ld_colors, float* radius, void* stream) {
    const char* what = "emer_flow_vis_color";
    EMER_REQUIRE(n >= 0, "%s: negative size", what);
    EMER_REQUIRE(scale_mode >= FLOW_SCALE_NONE && scale_mode <= FLOW_SCALE_DEVICE, "%s: scale mode %d", what,
                 scale_mode);
    if (n == 0) return 0;
    EMER_REQUIRE(flow && ld_flow >= 2, "%s: flow rows", what);
    EMER_REQUIRE(colors || radius, "%s: neither colours nor radii to write", what);
    EMER_REQUIRE(!colors || ld_colors >= 3, "%s: colour row stride %lld", what, (long long)ld_colors);
    EMER_REQUIRE(!colors || scale_mode != FLOW_SCALE_DEVICE || device_radius, "%s: NULL device radius", what);
    ColorParams p{};
    p.flow = flow; p.ld_flow = ld_flow; p.density = density; p.threshold = threshold; p.n = n;
    p.scale_mode = scale_mode;
    p.scale = 0.0f;
    if (scale_mode == FLOW_SCALE_HOST) p.scale = 1.0f / radius_scale;   // torch's CUDA division by a host scalar
    p.device_radius = device_radius; p.bright = bright != 0;
    p.colors = colors; p.ld_colors = ld_colors; p.radius = radius;
    flow_vis_color_kernel<<<(int)ceil_div(n, FV_THREADS), FV_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch(what);
}
