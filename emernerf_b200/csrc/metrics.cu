// The evaluation metrics of the reference, computed where the images live: one launch per image for the whole metric
// block of radiance_fields/video_utils.py:205-247 (PSNR, skimage's SSIM, their masked forms and the feature PSNRs), one
// for compute_valid_depth_rmse and one for compute_scene_flow_metrics (datasets/metrics.py:12-28, :73-128).  The
// reference copies both images to the host for two float32 SSIMs on one core and syncs on every boolean index; here
// every result lands in a caller-owned device array with no host sync.
//
// SSIM follows skimage.metrics.structural_similarity(data_range=1, channel_axis=-1) with its defaults: a 7 x 7 uniform
// window (scipy.ndimage.uniform_filter, 'reflect' border: d c b a | a b c d), sample covariance (49/48),
// C1 = 0.01^2, C2 = 0.03^2.  The five window moments and S are fp64: uxx - ux^2 cancels badly in fp32 when the variance
// is small next to C2, and the kernel is bound by its image reads, not by the arithmetic.
//
// Reduction: per-CTA fp64 partials go to the caller's workspace, and the CTA that takes the last ticket sums them in CTA
// order, writes the results and resets the ticket.  No float atomics: the same inputs on the same device give
// bit-identical results.
#include <math.h>

#include "common.cuh"
#include "cta_reduce.cuh"

namespace emer {

constexpr int MET_THREADS = 256;
constexpr int MET_WARPS = MET_THREADS / 32;
constexpr int MET_MAX_CTAS = 1024;
constexpr int MET_R = 3;                          // window radius (7 x 7)
constexpr int MET_TW = 32, MET_TH = 8;            // output tile: one pixel per thread in the vertical pass
constexpr int MET_SW = MET_TW + 2 * MET_R, MET_SH = MET_TH + 2 * MET_R;
constexpr int MET_MAX_C = 4;
constexpr int MET_MAX_CF = 256;
constexpr int MET_FEAT_UNROLL = 4;                // feature rows in flight per warp
static_assert(MET_TW * MET_TH == MET_THREADS, "one output pixel per thread");

// per-CTA partial sums (fp64) and extrema (fp32, NaN-propagating)
enum { P_SSE, P_MSSE, P_SSIM, P_MSSIM, P_FSSE, P_MFSSE, P_COUNT, P_N };
enum { E_XMIN, E_XMAX, E_YMIN, E_YMAX, E_N };

struct MetricsWorkspace {
    unsigned int ticket;                      // zero between calls: the last CTA resets it
    unsigned int pad[15];
    double sum[P_N][MET_MAX_CTAS];
    float ext[E_N][MET_MAX_CTAS];
};
static_assert(sizeof(MetricsWorkspace) <= EMER_METRICS_WORKSPACE_BYTES, "workspace layout exceeds the ABI size");

struct Partials {
    double s[P_N];
    float e[E_N];
};

__device__ __forceinline__ float nan_min(float a, float b) { return a != a ? a : (b != b ? b : fminf(a, b)); }
__device__ __forceinline__ float nan_max(float a, float b) { return a != a ? a : (b != b ? b : fmaxf(a, b)); }

__device__ __forceinline__ void init(Partials& p) {
#pragma unroll
    for (int k = 0; k < P_N; ++k) p.s[k] = 0.0;
    p.e[E_XMIN] = p.e[E_YMIN] = INFINITY;
    p.e[E_XMAX] = p.e[E_YMAX] = -INFINITY;
}

__device__ __forceinline__ void combine(Partials& a, const double* s, const float* e) {
#pragma unroll
    for (int k = 0; k < P_N; ++k) a.s[k] += s[k];
    a.e[E_XMIN] = nan_min(a.e[E_XMIN], e[E_XMIN]);
    a.e[E_XMAX] = nan_max(a.e[E_XMAX], e[E_XMAX]);
    a.e[E_YMIN] = nan_min(a.e[E_YMIN], e[E_YMIN]);
    a.e[E_YMAX] = nan_max(a.e[E_YMAX], e[E_YMAX]);
}

// Partials of one CTA in a fixed order (warp tree, then warps in index order); valid in thread 0.
__device__ void block_reduce(Partials& p) {
    __shared__ double shs[MET_WARPS][P_N];
    __shared__ float she[MET_WARPS][E_N];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        double s[P_N];
        float e[E_N];
#pragma unroll
        for (int k = 0; k < P_N; ++k) s[k] = __shfl_xor_sync(0xffffffffu, p.s[k], o);
#pragma unroll
        for (int k = 0; k < E_N; ++k) e[k] = __shfl_xor_sync(0xffffffffu, p.e[k], o);
        combine(p, s, e);
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) {
#pragma unroll
        for (int k = 0; k < P_N; ++k) shs[wid][k] = p.s[k];
#pragma unroll
        for (int k = 0; k < E_N; ++k) she[wid][k] = p.e[k];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        init(p);
        for (int w = 0; w < MET_WARPS; ++w) combine(p, shs[w], she[w]);
    }
}

// Every CTA publishes its partials; the one that takes the last ticket adds them up in CTA order.  Returns true in
// thread 0 of that CTA, with the totals in p.
__device__ bool reduce_across_ctas(Partials& p, MetricsWorkspace* ws) {
    block_reduce(p);
    if (threadIdx.x == 0) {
#pragma unroll
        for (int k = 0; k < P_N; ++k) ws->sum[k][blockIdx.x] = p.s[k];
#pragma unroll
        for (int k = 0; k < E_N; ++k) ws->ext[k][blockIdx.x] = p.e[k];
    }
    if (!take_last_ticket(&ws->ticket)) return false;
    init(p);
    for (int i = threadIdx.x; i < (int)gridDim.x; i += MET_THREADS) {
        double s[P_N];
        float e[E_N];
#pragma unroll
        for (int k = 0; k < P_N; ++k) s[k] = __ldcg(ws->sum[k] + i);
#pragma unroll
        for (int k = 0; k < E_N; ++k) e[k] = __ldcg(ws->ext[k] + i);
        combine(p, s, e);
    }
    block_reduce(p);
    release_ticket(&ws->ticket);
    return threadIdx.x == 0;
}

__device__ __forceinline__ double psnr_of(double sse, double count) { return -10.0 * log10(sse / count); }

// ---------------------------------------------------------------------------------------------- one image
struct ImageParams {
    const float* x;          // prediction [H, W, C]
    const float* y;          // target [H, W, C]
    const float* mask;       // [H, W] or null; nonzero = in the mask
    const float* fx;         // features [H * W rows, cf] with row strides ld_fx / ld_fy, or null
    const float* fy;
    int64_t ld_fx, ld_fy;
    int64_t h, w;
    int c, cf;
    int tiles_x, n_tiles, tile_ctas, feat_ctas;
    double* out;
    MetricsWorkspace* ws;
};

// scipy.ndimage 'reflect' (d c b a | a b c d) for indices within one window radius of the edge; clamped beyond that
// (the rows and columns of a partial tile that no output pixel reads)
__device__ __forceinline__ int64_t reflect(int64_t i, int64_t n) {
    if (i < 0) i = -i - 1;
    if (i >= n) i = 2 * n - i - 1;
    return i < 0 ? 0 : i;
}

__device__ void image_tiles(const ImageParams& p, Partials& acc) {
    __shared__ float sx[MET_SH][MET_SW * MET_MAX_C];
    __shared__ float sy[MET_SH][MET_SW * MET_MAX_C];
    __shared__ double hs[5][MET_SH][MET_TW];          // horizontal 7-sums of x, y, xx, yy, xy
    const int C = p.c, tid = threadIdx.x;
    const int ty = tid / MET_TW, tx = tid % MET_TW;
    const double cov = 49.0 / 48.0, c1 = 0.01 * 0.01, c2 = 0.03 * 0.03;
    for (int tile = blockIdx.x; tile < p.n_tiles; tile += p.tile_ctas) {
        const int64_t y0 = (int64_t)(tile / p.tiles_x) * MET_TH, x0 = (int64_t)(tile % p.tiles_x) * MET_TW;
        __syncthreads();                              // the previous tile's reads of sx / sy are done
        for (int i = tid; i < MET_SH * MET_SW * C; i += MET_THREADS) {
            const int r = i / (MET_SW * C), rem = i - r * (MET_SW * C);
            const int col = rem / C, ch = rem - col * C;
            const int64_t g = (reflect(y0 + r - MET_R, p.h) * p.w + reflect(x0 + col - MET_R, p.w)) * C + ch;
            sx[r][rem] = __ldg(p.x + g);
            sy[r][rem] = __ldg(p.y + g);
        }
        const int64_t gy = y0 + ty, gx = x0 + tx;
        const bool inside = gy < p.h && gx < p.w;
        const bool crop = inside && gy >= MET_R && gy < p.h - MET_R && gx >= MET_R && gx < p.w - MET_R;
        const bool masked = inside && p.mask && __ldg(p.mask + gy * p.w + gx) != 0.0f;
        if (masked) acc.s[P_COUNT] += 1.0;
        for (int ch = 0; ch < C; ++ch) {
            __syncthreads();                          // tile staged; the previous channel's reads of hs are done
            for (int i = tid; i < MET_SH * MET_TW; i += MET_THREADS) {
                const int r = i / MET_TW, j = i - r * MET_TW;
                double s1 = 0.0, s2 = 0.0, s11 = 0.0, s22 = 0.0, s12 = 0.0;
#pragma unroll
                for (int k = 0; k < 2 * MET_R + 1; ++k) {
                    const double a = sx[r][(j + k) * C + ch], b = sy[r][(j + k) * C + ch];
                    s1 += a; s2 += b;
                    s11 += a * a; s22 += b * b; s12 += a * b;
                }
                hs[0][r][j] = s1; hs[1][r][j] = s2; hs[2][r][j] = s11; hs[3][r][j] = s22; hs[4][r][j] = s12;
            }
            __syncthreads();
            if (!inside) continue;
            const float xv = sx[ty + MET_R][(tx + MET_R) * C + ch], yv = sy[ty + MET_R][(tx + MET_R) * C + ch];
            const double d = (double)xv - (double)yv;
            acc.s[P_SSE] += d * d;
            if (masked) acc.s[P_MSSE] += d * d;
            acc.e[E_XMIN] = nan_min(acc.e[E_XMIN], xv);
            acc.e[E_XMAX] = nan_max(acc.e[E_XMAX], xv);
            acc.e[E_YMIN] = nan_min(acc.e[E_YMIN], yv);
            acc.e[E_YMAX] = nan_max(acc.e[E_YMAX], yv);
            double m[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll
            for (int k = 0; k < 2 * MET_R + 1; ++k)
#pragma unroll
                for (int q = 0; q < 5; ++q) m[q] += hs[q][ty + k][tx];
            const double ux = m[0] / 49.0, uy = m[1] / 49.0, uxx = m[2] / 49.0, uyy = m[3] / 49.0, uxy = m[4] / 49.0;
            const double vx = cov * (uxx - ux * ux), vy = cov * (uyy - uy * uy), vxy = cov * (uxy - ux * uy);
            const double a1 = 2.0 * ux * uy + c1, a2 = 2.0 * vxy + c2;
            const double b1 = ux * ux + uy * uy + c1, b2 = vx + vy + c2;
            const double s = (a1 * a2) / (b1 * b2);
            if (crop) acc.s[P_SSIM] += s;
            if (masked) acc.s[P_MSSIM] += s;
        }
    }
}

// squared feature error per pixel row, one warp per row, MET_FEAT_UNROLL rows in flight
__device__ void feature_rows(const ImageParams& p, Partials& acc) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int64_t npix = p.h * p.w, nw = (int64_t)p.feat_ctas * MET_WARPS;
    for (int64_t r0 = (int64_t)(blockIdx.x - p.tile_ctas) * MET_WARPS + wid; r0 < npix; r0 += MET_FEAT_UNROLL * nw) {
        double e[MET_FEAT_UNROLL];
#pragma unroll
        for (int k = 0; k < MET_FEAT_UNROLL; ++k) e[k] = 0.0;
        for (int ch = lane; ch < p.cf; ch += 32) {
            float a[MET_FEAT_UNROLL], b[MET_FEAT_UNROLL];
#pragma unroll
            for (int k = 0; k < MET_FEAT_UNROLL; ++k) {
                const int64_t r = r0 + k * nw;
                a[k] = r < npix ? __ldg(p.fx + r * p.ld_fx + ch) : 0.0f;
                b[k] = r < npix ? __ldg(p.fy + r * p.ld_fy + ch) : 0.0f;
            }
#pragma unroll
            for (int k = 0; k < MET_FEAT_UNROLL; ++k) {
                const double d = (double)a[k] - (double)b[k];
                e[k] += d * d;
            }
        }
#pragma unroll
        for (int k = 0; k < MET_FEAT_UNROLL; ++k) {
            const int64_t r = r0 + k * nw;
            if (r >= npix) continue;
            acc.s[P_FSSE] += e[k];
            if (p.mask && __ldg(p.mask + r) != 0.0f) acc.s[P_MFSSE] += e[k];
        }
    }
}

__global__ void __launch_bounds__(MET_THREADS) image_metrics_kernel(const ImageParams p) {
    Partials acc;
    init(acc);
    if ((int)blockIdx.x < p.tile_ctas) image_tiles(p, acc);
    else feature_rows(p, acc);
    if (!reduce_across_ctas(acc, p.ws)) return;
    const double nan = __longlong_as_double(0x7ff8000000000000ll);
    const double pixels = (double)p.h * (double)p.w, count = acc.s[P_COUNT];
    const bool any = p.mask && count > 0.0;
    const bool feats = p.fx != nullptr;
    double* o = p.out;
    o[EMER_METRIC_PSNR] = psnr_of(acc.s[P_SSE], pixels * p.c);
    o[EMER_METRIC_SSIM] = acc.s[P_SSIM] / ((double)(p.h - 2 * MET_R) * (double)(p.w - 2 * MET_R) * p.c);
    o[EMER_METRIC_MASKED_PSNR] = any ? psnr_of(acc.s[P_MSSE], count * p.c) : nan;
    o[EMER_METRIC_MASKED_SSIM] = any ? acc.s[P_MSSIM] / (count * p.c) : nan;
    o[EMER_METRIC_FEAT_PSNR] = feats ? psnr_of(acc.s[P_FSSE], pixels * p.cf) : nan;
    o[EMER_METRIC_MASKED_FEAT_PSNR] = feats && any ? psnr_of(acc.s[P_MFSSE], count * p.cf) : nan;
    o[EMER_METRIC_MASK_COUNT] = p.mask ? count : nan;
    o[EMER_METRIC_PRED_MIN] = acc.e[E_XMIN];
    o[EMER_METRIC_PRED_MAX] = acc.e[E_XMAX];
    o[EMER_METRIC_TARGET_MIN] = acc.e[E_YMIN];
    o[EMER_METRIC_TARGET_MAX] = acc.e[E_YMAX];
}

// ---------------------------------------------------------------------------------------------- depth RMSE
__global__ void __launch_bounds__(MET_THREADS) depth_rmse_kernel(const float* pred, const float* target, int64_t n,
                                                               double* out, MetricsWorkspace* ws) {
    Partials acc;
    init(acc);
    for (int64_t i = (int64_t)blockIdx.x * MET_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * MET_THREADS) {
        const float t = __ldg(target + i);
        const double d = (double)__ldg(pred + i) - (double)t;
        acc.s[0] += d * d;
        if (t > 0.0f) { acc.s[1] += d * d; acc.s[2] += 1.0; }
    }
    if (!reduce_across_ctas(acc, ws)) return;
    out[0] = sqrt(acc.s[1] / acc.s[2]);          // NaN over no valid ray, as F.mse_loss of empty tensors
    out[1] = acc.s[2];
    out[2] = psnr_of(acc.s[0], (double)n);
}

// ---------------------------------------------------------------------------------------------- scene flow
// torch clamps with the bounds rounded to the tensor's dtype: +-(1 - 1e-7) in fp32
constexpr double FLOW_DOT_MAX = (double)(float)(1.0 - 1e-7);

__global__ void __launch_bounds__(MET_THREADS) scene_flow_kernel(const float* pred, const float* labels, int64_t n,
                                                               double* out, MetricsWorkspace* ws) {
    Partials acc;
    init(acc);
    for (int64_t i = (int64_t)blockIdx.x * MET_THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * MET_THREADS) {
        const double px = __ldg(pred + 3 * i), py = __ldg(pred + 3 * i + 1), pz = __ldg(pred + 3 * i + 2);
        const double lx = __ldg(labels + 3 * i), ly = __ldg(labels + 3 * i + 1), lz = __ldg(labels + 3 * i + 2);
        const double dx = px - lx, dy = py - ly, dz = pz - lz;
        const double l2 = sqrt(dx * dx + dy * dy + dz * dz);
        const double ln = sqrt(lx * lx + ly * ly + lz * lz);
        const double rel = l2 / (ln + 1e-20);
        acc.s[0] += l2;
        acc.s[1] += (l2 < 0.05 || rel < 0.05) ? 1.0 : 0.0;
        acc.s[2] += (l2 < 0.1 || rel < 0.1) ? 1.0 : 0.0;
        acc.s[3] += (l2 > 0.3 || rel > 0.1) ? 1.0 : 0.0;
        if (ln > 0.1) {
            const double pn = sqrt(px * px + py * py + pz * pz);
            const double dl = ln + 1e-7, dp = pn + 1e-7;         // unit vectors as the reference forms them
            double dot = (lx / dl) * (px / dp) + (ly / dl) * (py / dp) + (lz / dl) * (pz / dp);
            dot = dot != dot ? 0.0 : fmin(fmax(dot, -FLOW_DOT_MAX), FLOW_DOT_MAX);
            acc.s[4] += acos(dot);
            acc.s[5] += 1.0;
        }
    }
    if (!reduce_across_ctas(acc, ws)) return;
    const double m = (double)n;
    out[0] = acc.s[0] / m;
    out[1] = acc.s[1] / m;
    out[2] = acc.s[2] / m;
    out[3] = acc.s[3] / m;
    out[4] = acc.s[4] / acc.s[5];                // NaN when no label norm exceeds 0.1
    out[5] = acc.s[5];
    out[6] = m;
}

static int metrics_grid(int64_t work_items, int per_cta, int per_sm) {
    int64_t blocks = ceil_div(work_items, per_cta);
    int64_t cap = (int64_t)sm_count() * per_sm;
    if (cap > MET_MAX_CTAS / 2) cap = MET_MAX_CTAS / 2;
    if (blocks > cap) blocks = cap;
    return blocks < 1 ? 1 : (int)blocks;
}

}  // namespace emer

using namespace emer;

extern "C" int emer_image_metrics(const float* pred, const float* target, int64_t height, int64_t width, int channels,
                                  const float* mask, const float* feat_pred, int64_t ld_feat_pred,
                                  const float* feat_target, int64_t ld_feat_target, int feat_channels, double* out,
                                  void* workspace, void* stream) {
    EMER_REQUIRE(pred && target && out && workspace, "emer_image_metrics: NULL pointer");
    EMER_REQUIRE(channels >= 1 && channels <= MET_MAX_C, "emer_image_metrics: %d channels (1..%d)", channels, MET_MAX_C);
    EMER_REQUIRE(height >= 2 * MET_R + 1 && width >= 2 * MET_R + 1,
                 "emer_image_metrics: %lldx%lld image is smaller than the 7x7 SSIM window", (long long)height,
                 (long long)width);
    EMER_REQUIRE(!feat_pred == !feat_target, "emer_image_metrics: one feature map without the other");
    if (feat_pred) {
        EMER_REQUIRE(feat_channels >= 1 && feat_channels <= MET_MAX_CF, "emer_image_metrics: %d feature channels (1..%d)",
                     feat_channels, MET_MAX_CF);
        EMER_REQUIRE(ld_feat_pred >= feat_channels && ld_feat_target >= feat_channels,
                     "emer_image_metrics: feature row stride below the channel count");
    }
    ImageParams p{};
    p.x = pred; p.y = target; p.mask = mask;
    p.fx = feat_pred; p.fy = feat_target; p.ld_fx = ld_feat_pred; p.ld_fy = ld_feat_target;
    p.h = height; p.w = width; p.c = channels; p.cf = feat_pred ? feat_channels : 0;
    p.tiles_x = (int)ceil_div(width, MET_TW);
    const int64_t tiles = (int64_t)p.tiles_x * ceil_div(height, MET_TH);
    EMER_REQUIRE(tiles < (1ll << 31), "emer_image_metrics: image too large");
    p.n_tiles = (int)tiles;
    p.tile_ctas = metrics_grid(tiles, 1, 4);
    p.feat_ctas = feat_pred ? metrics_grid(height * width, MET_WARPS * MET_FEAT_UNROLL, 4) : 0;
    p.out = out;
    p.ws = (MetricsWorkspace*)workspace;
    image_metrics_kernel<<<p.tile_ctas + p.feat_ctas, MET_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_image_metrics");
}

extern "C" int emer_depth_rmse(const float* pred, const float* target, int64_t n, double* out, void* workspace,
                               void* stream) {
    EMER_REQUIRE(pred && target && out && workspace, "emer_depth_rmse: NULL pointer");
    EMER_REQUIRE(n >= 0, "emer_depth_rmse: negative size");
    depth_rmse_kernel<<<metrics_grid(n, MET_THREADS, 2), MET_THREADS, 0, (cudaStream_t)stream>>>(
        pred, target, n, out, (MetricsWorkspace*)workspace);
    return check_launch("emer_depth_rmse");
}

extern "C" int emer_scene_flow_metrics(const float* pred, const float* labels, int64_t n, double* out, void* workspace,
                                       void* stream) {
    EMER_REQUIRE(pred && labels && out && workspace, "emer_scene_flow_metrics: NULL pointer");
    EMER_REQUIRE(n >= 0, "emer_scene_flow_metrics: negative size");
    scene_flow_kernel<<<metrics_grid(n, MET_THREADS, 2), MET_THREADS, 0, (cudaStream_t)stream>>>(
        pred, labels, n, out, (MetricsWorkspace*)workspace);
    return check_launch("emer_scene_flow_metrics");
}
