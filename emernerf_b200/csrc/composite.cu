// Volume rendering along rays: transmittance / alpha / weights, opacity, expected and median
// depth, the proposal CDF, and weighted accumulation of per-sample values -- forward and
// backward.  Replaces nerfacc's batched render_transmittance_from_density /
// render_weight_from_density / accumulate_along_rays plus the torch cumsum / searchsorted /
// gather chain of radiance_fields/render_utils.py:73-115 and the CDF construction of
// third_party/nerfacc_prop_net.py:165-168.
//
// Layout: [R, S] row-major per-sample tensors; one warp per ray, lanes stride the samples
// (coalesced 128-byte rows), warp-shuffle scans carry the running sums between 32-sample
// chunks.  HBM-bound: ~ (3 reads + 2..3 writes) * 4 B per sample.
#include "common.cuh"
#include "ray_scan.cuh"

namespace emer {

constexpr int WARPS_PER_CTA = 8;

__global__ void __launch_bounds__(WARPS_PER_CTA * 32) composite_fwd_kernel(
    const float* __restrict__ t0, const float* __restrict__ t1, const float* __restrict__ sigma,
    float* __restrict__ weights, float* __restrict__ trans, float* __restrict__ opacity,
    float* __restrict__ depth, float* __restrict__ median, float* __restrict__ cdf, int64_t n_rays,
    int S) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (ray >= n_rays) return;
    const int64_t base = ray * S;
    RayScan<true> scan;
    for (int s0 = 0; s0 < S; s0 += 32) {
        const int s = s0 + lane;
        const bool ok = s < S;
        float a = 0.0f, b = 0.0f, sg = 0.0f;
        if (ok) {
            a = __ldg(t0 + base + s);
            b = __ldg(t1 + base + s);
            sg = __ldg(sigma + base + s);
        }
        float T;
        const float w = scan.step(a, b, sg, ok, s0, S, lane, T);
        if (ok) {
            if (weights) weights[base + s] = w;
            if (trans) trans[base + s] = T;
            if (cdf) cdf[ray * (S + 1) + s] = 1.0f - T;
        }
    }
    float op, dep, med;
    scan.finish(op, dep, med);
    if (lane == 0) {
        if (opacity) opacity[ray] = op;
        if (depth) depth[ray] = dep;
        if (median) median[ray] = med;
        if (cdf) cdf[ray * (S + 1) + S] = 1.0f;     // 1 - cat(trans, 0)[-1]
    }
}

// dL/dsigma from gradients on weights / trans / opacity / depth.
//   x_i = sigma_i*delta_i, T_i = exp(-sum_{j<i} x_j), w_i = T_i (1 - exp(-x_i))
//   G_i = g_w_i + g_opraw + g_D * mid_i           (total gradient reaching w_i)
//   dL/dx_i = G_i * T_i * exp(-x_i) - sum_{k>i} (G_k * w_k + g_T_k * T_k)
__global__ void __launch_bounds__(WARPS_PER_CTA * 32) composite_bwd_kernel(
    const float* __restrict__ t0, const float* __restrict__ t1, const float* __restrict__ sigma,
    const float* __restrict__ weights, const float* __restrict__ trans,
    const float* __restrict__ g_weights, const float* __restrict__ g_trans,
    const float* __restrict__ g_opacity, const float* __restrict__ g_depth,
    float* __restrict__ dsigma, int64_t n_rays, int S) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (ray >= n_rays) return;
    const int64_t base = ray * S;
    // pass 1: ray totals
    float sum_w = 0.0f, sum_wm = 0.0f;
    for (int s = lane; s < S; s += 32) {
        const float w = __ldg(weights + base + s);
        const float mid = (__ldg(t0 + base + s) + __ldg(t1 + base + s)) / 2.0f;
        sum_w += w;
        sum_wm = fmaf(w, mid, sum_wm);
    }
    sum_w = warp_sum(sum_w);
    sum_wm = warp_sum(sum_wm);
    const float op = fminf(fmaxf(sum_w, 1e-6f), 1.0f);
    const float gd = g_depth ? __ldg(g_depth + ray) : 0.0f;
    const float go = g_opacity ? __ldg(g_opacity + ray) : 0.0f;
    const float g_D = gd / op;                                   // depth = D / op
    float g_op = go - gd * sum_wm / (op * op);
    const float g_opraw = (sum_w >= 1e-6f && sum_w <= 1.0f) ? g_op : 0.0f;   // clamp passes in range
    // pass 2: reverse sweep with a running suffix sum
    float carry = 0.0f;
    const int chunks = (S + 31) / 32;
    for (int ch = chunks - 1; ch >= 0; --ch) {
        const int s = ch * 32 + lane;
        const bool ok = s < S;
        float a = 0.0f, b = 0.0f, sg = 0.0f, w = 0.0f, T = 0.0f, gw = 0.0f, gT = 0.0f;
        if (ok) {
            a = __ldg(t0 + base + s);
            b = __ldg(t1 + base + s);
            sg = __ldg(sigma + base + s);
            w = __ldg(weights + base + s);
            T = __ldg(trans + base + s);
            if (g_weights) gw = __ldg(g_weights + base + s);
            if (g_trans) gT = __ldg(g_trans + base + s);
        }
        const float delta = b - a;
        const float mid = (a + b) / 2.0f;
        const float G = gw + g_opraw + g_D * mid;
        const float q = ok ? fmaf(G, w, gT * T) : 0.0f;
        const float suf_incl = warp_scan_incl_rev(q, lane);
        const float suffix_excl = carry + (suf_incl - q);
        const float ex = expf(-(sg * delta));
        const float dx = G * T * ex - suffix_excl;
        if (ok) dsigma[base + s] = dx * delta;
        carry += __shfl_sync(0xffffffffu, suf_incl, 0);
    }
}

// out[R, C] = sum_s w[R,S] * v[R,S,C].  One warp per ray.
// C <= 4: lanes stride the samples, shuffle-reduce.  Otherwise lanes stride the channels.
template <int C>
__global__ void __launch_bounds__(WARPS_PER_CTA * 32) accumulate_small_fwd_kernel(
    const float* __restrict__ w, const float* __restrict__ v, float* __restrict__ out, int64_t n_rays, int S) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (ray >= n_rays) return;
    float acc[C];
#pragma unroll
    for (int c = 0; c < C; ++c) acc[c] = 0.0f;
    for (int s = lane; s < S; s += 32) {
        const float ws = __ldg(w + ray * S + s);
        const float* vp = v + (ray * S + s) * C;
#pragma unroll
        for (int c = 0; c < C; ++c) acc[c] = fmaf(ws, __ldg(vp + c), acc[c]);
    }
#pragma unroll
    for (int c = 0; c < C; ++c) {
        const float t = warp_sum(acc[c]);
        if (lane == 0) out[ray * C + c] = t;
    }
}

constexpr int ACC_MAX_PER_LANE = 8;   // C <= 256
__global__ void __launch_bounds__(WARPS_PER_CTA * 32) accumulate_wide_fwd_kernel(
    const float* __restrict__ w, const float* __restrict__ v, float* __restrict__ out, int64_t n_rays, int S,
    int C) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (ray >= n_rays) return;
    float acc[ACC_MAX_PER_LANE];
#pragma unroll
    for (int j = 0; j < ACC_MAX_PER_LANE; ++j) acc[j] = 0.0f;
    for (int s = 0; s < S; ++s) {
        const float ws = __ldg(w + ray * S + s);
        const float* vp = v + (ray * S + s) * (int64_t)C;
#pragma unroll
        for (int j = 0; j < ACC_MAX_PER_LANE; ++j) {
            const int c = lane + j * 32;
            if (c < C) acc[j] = fmaf(ws, __ldg(vp + c), acc[j]);
        }
    }
#pragma unroll
    for (int j = 0; j < ACC_MAX_PER_LANE; ++j) {
        const int c = lane + j * 32;
        if (c < C) out[ray * C + c] = acc[j];
    }
}

// dw[r,s] = sum_c g[r,c] v[r,s,c];  dv[r,s,c] = w[r,s] g[r,c].   One thread per (r, s) for small C,
// one warp per (r, s) otherwise.
__global__ void accumulate_bwd_small_kernel(const float* __restrict__ w, const float* __restrict__ v,
                                            const float* __restrict__ g, float* __restrict__ dw,
                                            float* __restrict__ dv, int64_t total, int S, int C) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int64_t ray = i / S;
    const float ws = dv ? __ldg(w + i) : 0.0f;
    float acc = 0.0f;
    for (int c = 0; c < C; ++c) {
        const float gc = __ldg(g + ray * C + c);
        if (dw) acc = fmaf(gc, __ldg(v + i * C + c), acc);
        if (dv) dv[i * C + c] = ws * gc;
    }
    if (dw) dw[i] = acc;
}

__global__ void __launch_bounds__(WARPS_PER_CTA * 32) accumulate_bwd_wide_kernel(
    const float* __restrict__ w, const float* __restrict__ v, const float* __restrict__ g,
    float* __restrict__ dw, float* __restrict__ dv, int64_t total, int S, int C) {
    const int lane = threadIdx.x & 31;
    const int64_t i = (int64_t)blockIdx.x * WARPS_PER_CTA + (threadIdx.x >> 5);
    if (i >= total) return;
    const int64_t ray = i / S;
    const float ws = dv ? __ldg(w + i) : 0.0f;
    float acc = 0.0f;
    for (int c = lane; c < C; c += 32) {
        const float gc = __ldg(g + ray * C + c);
        if (dw) acc = fmaf(gc, __ldg(v + i * C + c), acc);
        if (dv) dv[i * C + c] = ws * gc;
    }
    if (dw) {
        acc = warp_sum(acc);
        if (lane == 0) dw[i] = acc;
    }
}

}  // namespace emer

using namespace emer;

extern "C" int emer_composite_fwd(const float* t0, const float* t1, const float* sigma, float* weights,
                                  float* trans, float* opacity, float* depth, float* median_depth, float* cdf,
                                  int64_t n_rays, int n_samples, void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(t0 && t1 && sigma, "emer_composite_fwd: NULL pointer");
    EMER_REQUIRE(n_samples >= 1, "emer_composite_fwd: n_samples must be >= 1");
    composite_fwd_kernel<<<(unsigned)ceil_div(n_rays, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, (cudaStream_t)stream>>>(
        t0, t1, sigma, weights, trans, opacity, depth, median_depth, cdf, n_rays, n_samples);
    return check_launch("emer_composite_fwd");
}

extern "C" int emer_composite_bwd(const float* t0, const float* t1, const float* sigma, const float* weights,
                                  const float* trans, const float* g_weights, const float* g_trans,
                                  const float* g_opacity, const float* g_depth, float* dsigma, int64_t n_rays,
                                  int n_samples, void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(t0 && t1 && sigma && weights && trans && dsigma, "emer_composite_bwd: NULL pointer");
    composite_bwd_kernel<<<(unsigned)ceil_div(n_rays, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, (cudaStream_t)stream>>>(
        t0, t1, sigma, weights, trans, g_weights, g_trans, g_opacity, g_depth, dsigma, n_rays, n_samples);
    return check_launch("emer_composite_bwd");
}

extern "C" int emer_accumulate_fwd(const float* w, const float* v, float* out, int64_t n_rays, int n_samples,
                                   int c, void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(w && v && out, "emer_accumulate_fwd: NULL pointer");
    EMER_REQUIRE(c >= 1 && c <= 32 * ACC_MAX_PER_LANE, "emer_accumulate_fwd: channels %d out of range", c);
    const unsigned blocks = (unsigned)ceil_div(n_rays, WARPS_PER_CTA);
    const int threads = WARPS_PER_CTA * 32;
    cudaStream_t st = (cudaStream_t)stream;
    switch (c) {
        case 1: accumulate_small_fwd_kernel<1><<<blocks, threads, 0, st>>>(w, v, out, n_rays, n_samples); break;
        case 2: accumulate_small_fwd_kernel<2><<<blocks, threads, 0, st>>>(w, v, out, n_rays, n_samples); break;
        case 3: accumulate_small_fwd_kernel<3><<<blocks, threads, 0, st>>>(w, v, out, n_rays, n_samples); break;
        case 4: accumulate_small_fwd_kernel<4><<<blocks, threads, 0, st>>>(w, v, out, n_rays, n_samples); break;
        default: accumulate_wide_fwd_kernel<<<blocks, threads, 0, st>>>(w, v, out, n_rays, n_samples, c);
    }
    return check_launch("emer_accumulate_fwd");
}

extern "C" int emer_accumulate_bwd(const float* w, const float* v, const float* g, float* dw, float* dv,
                                   int64_t n_rays, int n_samples, int c, void* stream) {
    if (n_rays == 0 || (!dw && !dv)) return 0;
    EMER_REQUIRE(w && v && g, "emer_accumulate_bwd: NULL pointer");
    const int64_t total = n_rays * n_samples;
    cudaStream_t st = (cudaStream_t)stream;
    if (c <= 8) {
        accumulate_bwd_small_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, st>>>(w, v, g, dw, dv, total, n_samples, c);
    } else {
        accumulate_bwd_wide_kernel<<<(unsigned)ceil_div(total, WARPS_PER_CTA), WARPS_PER_CTA * 32, 0, st>>>(
            w, v, g, dw, dv, total, n_samples, c);
    }
    return check_launch("emer_accumulate_bwd");
}
