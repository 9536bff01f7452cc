// The evaluation video frames of the reference's save_videos (radiance_fields/video_utils.py:471-627).  The reference
// keeps every product of every image as a float32 numpy array until all images are rendered, then per frame colours
// the depths on the host (visualize_depth: float64 log curve and a matplotlib turbo lookup), blends, concatenates in
// float64 and applies to8b.  Here each image's products stay on the device:
//
// emer_video_compose: one launch per image.  Block (x, t) handles pixels x * VID_THREADS.. of tile t, one thread per
//   pixel: it reads the tile's inputs, applies the tile's kind (csrc/video.cuh) and writes three bytes into the
//   image's column of the tile's frame row.  Offsets are 64-bit; each thread checks its pixel against H * W.
#include "common.cuh"
#include "video.cuh"

namespace emer {

constexpr int VID_THREADS = 256;

struct VideoParams {
    emer_video_tile tiles[EMER_VIDEO_MAX_TILES];  // by value: no device copy of the descriptors, nothing to free
    uint8_t* frame;
    const uint8_t* lut;
    int64_t frame_w, height, width, pixels, col;
};

__global__ void __launch_bounds__(VID_THREADS) video_compose_kernel(const __grid_constant__ VideoParams p) {
    const int64_t px = (int64_t)blockIdx.x * VID_THREADS + threadIdx.x;
    if (px >= p.pixels) return;
    const emer_video_tile& t = p.tiles[blockIdx.y];
    const bool f64 = t.f64 != 0;
    uint8_t rgb[3];
    switch (t.kind) {
        case EMER_VIDEO_RGB:
#pragma unroll
            for (int c = 0; c < 3; ++c) rgb[c] = video_to8b(__ldg(t.in[0] + 3 * px + c), f64);
            break;
        case EMER_VIDEO_DEPTH: {
            const int i = video_depth_index(__ldg(t.in[0] + px), __ldg(t.in[1] + px));
#pragma unroll
            for (int c = 0; c < 3; ++c) rgb[c] = i < 0 ? (uint8_t)0 : __ldg(p.lut + 3 * i + c);
            break;
        }
        case EMER_VIDEO_BLEND: {
            const float alpha = __ldg(t.in[1] + px);
#pragma unroll
            for (int c = 0; c < 3; ++c)
                rgb[c] = video_to8b(video_blend(__ldg(t.in[0] + 3 * px + c), alpha, __ldg(t.in[2] + 3 * px + c)), f64);
            break;
        }
        default: {  // EMER_VIDEO_GRAY
            float v = __ldg(t.in[0] + px);
            if (t.invert) v = __fsub_rn(1.0f, v);
            rgb[0] = rgb[1] = rgb[2] = video_to8b(v, f64);
            break;
        }
    }
    const int64_t y = px / p.width, x = px - y * p.width;
    const int64_t o = (((int64_t)t.row * p.height + y) * p.frame_w + p.col * p.width + x) * 3;
    p.frame[o] = rgb[0];
    p.frame[o + 1] = rgb[1];
    p.frame[o + 2] = rgb[2];
}

}  // namespace emer

using namespace emer;

extern "C" int emer_video_compose(uint8_t* frame, int64_t frame_w, const emer_video_tile* tiles, int n_tiles,
                                  int64_t height, int64_t width, int col, const uint8_t* lut, void* stream) {
    const char* what = "emer_video_compose";
    EMER_REQUIRE(frame && tiles, "%s: NULL pointer", what);
    EMER_REQUIRE(n_tiles >= 1 && n_tiles <= EMER_VIDEO_MAX_TILES, "%s: %d tiles (1..%d)", what, n_tiles,
                 EMER_VIDEO_MAX_TILES);
    EMER_REQUIRE(height >= 1 && width >= 1 && height * width <= EMER_VIDEO_MAX_PIXELS, "%s: a %lld x %lld tile", what,
                 (long long)height, (long long)width);
    EMER_REQUIRE(col >= 0 && ((int64_t)col + 1) * width <= frame_w, "%s: column %d of %lld pixels in a frame %lld wide",
                 what, col, (long long)width, (long long)frame_w);
    VideoParams p{};
    for (int i = 0; i < n_tiles; ++i) {
        const emer_video_tile& t = tiles[i];
        EMER_REQUIRE(t.kind >= EMER_VIDEO_RGB && t.kind <= EMER_VIDEO_GRAY, "%s: tile %d of kind %d", what, i, t.kind);
        EMER_REQUIRE(t.row >= 0, "%s: tile %d at row %d", what, i, t.row);
        const int need = t.kind == EMER_VIDEO_BLEND ? 3 : t.kind == EMER_VIDEO_DEPTH ? 2 : 1;
        for (int k = 0; k < need; ++k) EMER_REQUIRE(t.in[k], "%s: tile %d lacks input %d", what, i, k);
        EMER_REQUIRE(t.kind != EMER_VIDEO_DEPTH || lut, "%s: a depth tile without the colour table", what);
        p.tiles[i] = t;
    }
    p.frame = frame; p.lut = lut; p.frame_w = frame_w; p.height = height; p.width = width;
    p.pixels = height * width; p.col = col;
    const dim3 grid((unsigned)ceil_div(p.pixels, VID_THREADS), (unsigned)n_tiles);
    video_compose_kernel<<<grid, VID_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch(what);
}
