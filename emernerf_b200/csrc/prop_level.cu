// One proposal level in ONE launch (no-grad path of PropNetEstimator.sampling):
//   inverse-CDF resampling of the previous level -> s->t warp -> ray march -> contraction+selector ->
//   hash grid (3-D, F floats x L levels <= 16 features) -> Linear(LF,64)-ReLU-Linear(64,1) ->
//   trunc_exp(x-1) -> sigma*delta -> exclusive scan along the ray -> CDF of this level, 1 - the running minimum of T
//   (the composite's monotone_trans, ray_scan.cuh: non-decreasing along every ray).
// Replaces, per level, ~15 launches of the modular path (third_party/nerfacc_prop_net.py:147-170 with
// render_utils.py:314-324 and radiance_field.py:825-841 of the reference) and every intermediate
// [R,S,*] tensor: the only HBM traffic is the table gathers (L2-resident: 18-22 MB tables) and the
// [R, n+1] edges / CDF rows.  Resampling, contraction and grid lookup are the device functions of emer_pdf_resample,
// emer_contract_fwd and emer_grid_fwd (sampling.cuh, contract.cuh, grid_common.cuh), so s/t edges, positions and table
// indices are bit-identical to the modular path's; the MLP runs on the FP32 FMA pipe with weights broadcast from
// shared memory.
//
// One warp per ray; lane l owns edges / samples l, l+32, ... (n <= 256).
#include "common.cuh"
#include "contract.cuh"
#include "grid_common.cuh"
#include "ray_scan.cuh"
#include "sampling.cuh"

namespace emer {

struct PropParams {
    emer_grid_desc g;
    const float* prev_s;      // [R, m1]
    const float* prev_cdf;    // [R, m1]
    const float* bias;        // [R] or null (0.5)
    const float* origins;     // [R, 3]
    const float* dirs;        // [R, 3]
    const float* aabb;        // [6]
    const float* table;
    const float* w0;          // [64, LF]
    const float* b0;          // [64]
    const float* w1;          // [64]
    const float* b1;          // [1]
    float* out_s;             // [R, n+1]
    float* out_t;             // [R, n+1]
    float* out_cdf;           // [R, n+1]
    float* out_sigma;         // [R, n] or null: the densities, kept for emer_prop_level_bwd
    int64_t n_rays;
    int m1, n, stot_kind, unbounded;
    float s_min, s_max;
};

constexpr int PL_WARPS = 8;
constexpr int PL_MAX_EDGES = 257;
constexpr int PL_HID = 64;
constexpr int PL_MAX_IN = 16;

// what a warp needs of its ray
struct PlRay {
    float ox, oy, oz, dx, dy, dz, lo3[3], hi3[3];
};

__device__ __forceinline__ PlRay pl_load_ray(const float* origins, const float* dirs, const float* aabb, int64_t ray) {
    PlRay rc;
    rc.ox = __ldg(origins + ray * 3); rc.oy = __ldg(origins + ray * 3 + 1); rc.oz = __ldg(origins + ray * 3 + 2);
    rc.dx = __ldg(dirs + ray * 3); rc.dy = __ldg(dirs + ray * 3 + 1); rc.dz = __ldg(dirs + ray * 3 + 2);
    load_box(aabb, rc.lo3, rc.hi3);
    return rc;
}

// Interval midpoint -> contracted, selector-masked grid coordinate xc -> hash-grid features enc.  ONE body for the
// forward and the backward kernel, so the backward re-derives bit for bit what the forward saw.  Called by all 32
// lanes of the warp (lanes past the ray's last sample repeat it): with LF_T > 0, lane pairs share the corner loads.
template <int LF_T>
__device__ __forceinline__ void pl_encode(const emer_grid_desc& g, const float* __restrict__ table, int unbounded,
                                          const PlRay& rc, float t0, float t1, float (&xc)[3],
                                          float (&enc)[LF_T > 0 ? LF_T : PL_MAX_IN]) {
    const int L = LF_T > 0 ? LF_T : g.n_levels, F = LF_T > 0 ? 1 : g.n_feat;
    const float tt = t0 + t1;
    // positions = origins + dirs * (t0 + t1) / 2   (render_utils.py:318)
    float pos[3] = {rc.ox + rc.dx * tt / 2.0f, rc.oy + rc.dy * tt / 2.0f, rc.oz + rc.dz * tt / 2.0f};
    float xn[3], mag;
    int amax;
    bool sel;
    contract_point(pos, rc.lo3, rc.hi3, unbounded, 1, xc, xn, mag, amax, sel);
    float xq[3];                                // the lane pair's other sample (LF_T > 0)
#pragma unroll
    for (int d = 0; d < 3; ++d) xq[d] = LF_T > 0 ? shfl_xor1(xc[d]) : 0.0f;
#pragma unroll
    for (int l = 0; l < L; ++l) {
        const uint32_t res = g.resolution[l], off = g.offset[l], size = g.offset[l + 1] - off;
        const bool hashed = g.hashed[l] != 0;
        uint32_t c0[3];
        float w[3];
        locate<3>(xc, g.scale[l], c0, w);
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        if constexpr (LF_T > 0) {
            // F = 1: the x-neighbour corners of a cell in one load instruction of a lane pair (gather_corner_pairs);
            // the same values, accumulated in the same order
            uint32_t c0q[3];
            float wq[3];
            locate<3>(xq, g.scale[l], c0q, wq);
            float val[8];
            gather_corner_pairs<3>(table + off, c0, c0q, res, size, hashed, val);
#pragma unroll
            for (int cc = 0; cc < 8; ++cc) acc[0] = fmaf(corner_weight<3>(cc, w), val[cc], acc[0]);
        } else {
#pragma unroll
            for (int cc = 0; cc < 8; ++cc) {
                const float wt = corner_weight<3>(cc, w);
                uint32_t ci[3];
                corner_cell<3>(cc, c0, ci);
                const float* e = table + ((size_t)off + grid_index<3>(ci, res, size, hashed)) * F;
                for (int f = 0; f < F; ++f) acc[f] = fmaf(wt, __ldg(e + f), acc[f]);
            }
        }
        if (LF_T > 0) enc[l] = acc[0];
        else for (int f = 0; f < F; ++f) enc[l * F + f] = acc[f];
    }
}

template <int LF>
__device__ __forceinline__ void pl_load_row(const float* __restrict__ row16, float (&w)[LF]) {     // 16-byte aligned
#pragma unroll
    for (int i = 0; i < LF; i += 4) {
        const float4 v = *reinterpret_cast<const float4*>(row16 + i);
        w[i] = v.x; w[i + 1] = v.y; w[i + 2] = v.z; w[i + 3] = v.w;
    }
}

// LF_T > 0: compile-time feature count with F = 1 (the shipped proposal grids: 8 levels x 1 feature);
// LF_T == 0: generic run-time loops.  Two CTAs per SM, as the ~100 registers allow: left to itself, ptxas squeezes
// <8> into 80 registers and spills.
template <int LF_T>
__global__ void __launch_bounds__(PL_WARPS * 32, 2) prop_level_kernel(const PropParams p) {
    __shared__ float t_edges[PL_WARPS][PL_MAX_EDGES + 3];
    __shared__ __align__(16) float w0s[PL_HID * PL_MAX_IN];
    __shared__ float b0s[PL_HID], w1s[PL_HID];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int LF = LF_T > 0 ? LF_T : p.g.n_levels * p.g.n_feat;
    for (int e = tid; e < PL_HID * LF; e += PL_WARPS * 32) w0s[e] = __ldg(p.w0 + e);
    for (int e = tid; e < PL_HID; e += PL_WARPS * 32) { b0s[e] = __ldg(p.b0 + e); w1s[e] = __ldg(p.w1 + e); }
    __syncthreads();
    const float b1 = __ldg(p.b1);
    const int64_t ray = (int64_t)blockIdx.x * PL_WARPS + wid;
    if (ray >= p.n_rays) return;
    const int n = p.n, m1 = p.m1;

    // ---- 1. inverse-CDF resampling
    const float bb = p.bias ? __ldg(p.bias + ray) : 0.5f;
    for (int k = lane; k <= n; k += 32) {
        int bin;
        const float s = resample_edge(p.prev_cdf + ray * m1, p.prev_s + ray * m1, m1, n, k, bb, bin);
        const float t = s_to_t(s, p.s_min, p.s_max, p.stot_kind);
        p.out_s[ray * (n + 1) + k] = s;
        p.out_t[ray * (n + 1) + k] = t;
        t_edges[wid][k] = t;
    }
    __syncwarp();

    // ---- 2. density at the interval midpoints, 3. scan -> CDF
    const PlRay rc = pl_load_ray(p.origins, p.dirs, p.aabb, ray);
    float carry = 0.0f, carry_t = 1.0f;
    for (int k0 = 0; k0 < n; k0 += 32) {
        const int k = k0 + lane;
        const bool ok = k < n;
        float xdelta = 0.0f;
        const int kc = ok ? k : n - 1;
        const float t0 = t_edges[wid][kc], t1 = t_edges[wid][kc + 1];
        float xc[3];
        float enc[LF_T > 0 ? LF_T : PL_MAX_IN];
        pl_encode<LF_T>(p.g, p.table, p.unbounded, rc, t0, t1, xc, enc);
        if (ok) {
            // Linear(LF, 64) - ReLU - Linear(64, 1) - trunc_exp(. - 1)
            float raw = b1;
#pragma unroll 4
            for (int j = 0; j < PL_HID; ++j) {
                float h = b0s[j];
#pragma unroll
                for (int i = 0; i < LF; ++i) h = fmaf(w0s[j * LF + i], enc[i], h);
                h = h > 0.0f ? h : 0.0f;
                raw = fmaf(w1s[j], h, raw);
            }
            const float sigma = density_fwd(raw);
            xdelta = sigma * (t1 - t0);
            if (p.out_sigma) p.out_sigma[ray * n + k] = sigma;
        }
        const float incl = warp_scan_incl(xdelta, lane);
        const float e_excl = carry + warp_scan_excl(incl, lane);
        const float T = monotone_trans(expf(-e_excl), carry_t, lane);    // the composite's CDF: never falls
        if (ok) p.out_cdf[ray * (n + 1) + k] = 1.0f - T;
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) p.out_cdf[ray * (n + 1) + n] = 1.0f;
}

// ---------------------------------------------------------------------------------------------------------------
// Backward of one proposal level (the steps on which the proposal networks are updated).
//
// The interlevel loss reaches a level only through its CDF row (the sample positions are drawn without gradient,
// third_party/nerfacc_prop_net.py:147-170 of the reference), so the whole backward is a function of d_cdf [R, n+1]:
//   cdf_k = 1 - exp(-E_k),  E_k = sum_{j<k} sigma_j delta_j       dE_k = d_cdf_k exp(-E_k)           (k < n)
//   d(sigma_j delta_j) = sum_{k>j} dE_k                           d_raw_j = that * delta_j * exp(min(raw_j - 1, 15))
//   raw = b1 + w1 . relu(W0 enc + b0)                             -> dW0, db0, dw1, db1, d_enc
// One warp per ray, persistent CTAs.  sigma comes from the forward (out_sigma); positions, grid features and hidden
// units are recomputed with the forward's own code (pl_encode), so no [N, 64] activation ever exists in HBM:
// the modular path wrote and re-read ~1.2 KB per sample for this, here it is 44 B (xc, d_enc for the grid scatter,
// which stays emer_grid_bwd).  Per 32 samples a warp works in two layouts:
//   lane = sample: h_j, relu mask, d_enc_i = sum_j dh_j W0[j][i]           (weights broadcast from shared memory)
//   lane = hidden unit (j = lane, lane + 32): the samples' enc / d_raw are broadcast by shuffles, the unit's
//     dW0 row, db0, dw1 accumulate in registers over every ray the warp owns and are flushed once per CTA.
struct PropBwdParams {
    emer_grid_desc g;
    const float* t_edges;     // [R, n+1]
    const float* sigma;       // [R, n]
    const float* d_cdf;       // [R, n+1]
    const float* origins;
    const float* dirs;
    const float* aabb;
    const float* table;
    const float* w0;
    const float* b0;
    const float* w1;
    float* xc;                // [R n, 3]   out: grid coordinates of the samples
    float* d_enc;             // [R n, LF]  out
    float* d_w0;              // [64, LF]   accumulated
    float* d_b0;              // [64]       accumulated
    float* d_w1;              // [64]       accumulated
    float* d_b1;              // [1]        accumulated
    int64_t n_rays;
    int n, unbounded;
};

template <int LF>
__global__ void __launch_bounds__(PL_WARPS * 32) prop_level_bwd_kernel(const PropBwdParams p) {
    __shared__ float t_edges[PL_WARPS][PL_MAX_EDGES + 3];
    __shared__ float d_raw_s[PL_WARPS][PL_MAX_EDGES + 3];
    __shared__ __align__(16) float w0s[PL_HID * LF];
    __shared__ float b0s[PL_HID], w1s[PL_HID];
    __shared__ float red[PL_HID * LF + 2 * PL_HID + 1];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    for (int e = tid; e < PL_HID * LF; e += PL_WARPS * 32) w0s[e] = __ldg(p.w0 + e);
    for (int e = tid; e < PL_HID; e += PL_WARPS * 32) { b0s[e] = __ldg(p.b0 + e); w1s[e] = __ldg(p.w1 + e); }
    for (int e = tid; e < PL_HID * LF + 2 * PL_HID + 1; e += PL_WARPS * 32) red[e] = 0.0f;
    __syncthreads();
    // unit layout: this lane's two hidden units
    float w0r[2][LF], b0r[2], w1r[2], acc_w0[2][LF], acc_b0[2], acc_w1[2];
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int j = lane + 32 * u;
#pragma unroll
        for (int i = 0; i < LF; ++i) { w0r[u][i] = w0s[j * LF + i]; acc_w0[u][i] = 0.0f; }
        b0r[u] = b0s[j]; w1r[u] = w1s[j]; acc_b0[u] = 0.0f; acc_w1[u] = 0.0f;
    }
    float acc_b1 = 0.0f;
    const int n = p.n;
    for (int64_t ray = (int64_t)blockIdx.x * PL_WARPS + wid; ray < p.n_rays; ray += (int64_t)gridDim.x * PL_WARPS) {
        __syncwarp();
        for (int k = lane; k <= n; k += 32) t_edges[wid][k] = __ldg(p.t_edges + ray * (n + 1) + k);
        __syncwarp();
        // ---- 1. forward scan again (same arithmetic as the forward) -> dE_k = d_cdf_k exp(-E_k)
        float carry = 0.0f;
        for (int k0 = 0; k0 < n; k0 += 32) {
            const int k = k0 + lane;
            const bool ok = k < n;
            float xdelta = 0.0f;
            if (ok) xdelta = __ldg(p.sigma + ray * n + k) * (t_edges[wid][k + 1] - t_edges[wid][k]);
            const float incl = warp_scan_incl(xdelta, lane);
            const float e_excl = carry + warp_scan_excl(incl, lane);   // bit-identical to the forward
            if (ok) d_raw_s[wid][k] = __ldg(p.d_cdf + ray * (n + 1) + k) * expf(-e_excl);
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        __syncwarp();
        // ---- 2. exclusive suffix sums, last chunk first -> d_raw_k (in place)
        float tail = 0.0f;
        for (int k0 = ((n - 1) / 32) * 32; k0 >= 0; k0 -= 32) {
            const int k = k0 + (31 - lane);            // lane 0 takes the chunk's LAST sample
            const bool ok = k < n;
            const float v = ok ? d_raw_s[wid][k] : 0.0f;
            const float incl = warp_scan_incl(v, lane);
            const float g_excl = tail + warp_scan_excl(incl, lane);    // sum over the samples behind k
            if (ok) {
                const float sg = __ldg(p.sigma + ray * n + k);
                d_raw_s[wid][k] = g_excl * (t_edges[wid][k + 1] - t_edges[wid][k]) * fminf(sg, 3269017.372472111f);   // e^15
            }
            tail += __shfl_sync(0xffffffffu, incl, 31);
        }
        __syncwarp();
        // ---- 3. per sample: encode again, MLP forward + backward
        const PlRay rc = pl_load_ray(p.origins, p.dirs, p.aabb, ray);
        for (int k0 = 0; k0 < n; k0 += 32) {
            const int k = k0 + lane;
            const bool ok = k < n;
            float enc[LF], d_enc[LF], xc[3] = {0.f, 0.f, 0.f};
            float d_raw = 0.0f;
#pragma unroll
            for (int i = 0; i < LF; ++i) { enc[i] = 0.0f; d_enc[i] = 0.0f; }
            const int kc = ok ? k : n - 1;
            pl_encode<LF>(p.g, p.table, p.unbounded, rc, t_edges[wid][kc], t_edges[wid][kc + 1], xc, enc);
            if (!ok) {
#pragma unroll
                for (int i = 0; i < LF; ++i) enc[i] = 0.0f;
            } else {
                d_raw = d_raw_s[wid][k];
#pragma unroll 4
                for (int j = 0; j < PL_HID; ++j) {
                    float h = b0s[j];
                    float wr[LF];
                    pl_load_row<LF>(w0s + j * LF, wr);
#pragma unroll
                    for (int i = 0; i < LF; ++i) h = fmaf(wr[i], enc[i], h);
                    const float dh = h > 0.0f ? d_raw * w1s[j] : 0.0f;
#pragma unroll
                    for (int i = 0; i < LF; ++i) d_enc[i] = fmaf(dh, wr[i], d_enc[i]);
                }
                const int64_t pt = ray * n + k;
                p.xc[pt * 3] = xc[0]; p.xc[pt * 3 + 1] = xc[1]; p.xc[pt * 3 + 2] = xc[2];
#pragma unroll
                for (int i = 0; i < LF; i += 4)
                    *reinterpret_cast<float4*>(p.d_enc + pt * LF + i) = make_float4(d_enc[i], d_enc[i + 1], d_enc[i + 2], d_enc[i + 3]);
                acc_b1 += d_raw;
            }
            // unit layout over the chunk's 32 samples (lanes past n carry enc = 0, d_raw = 0: no contribution)
            for (int sidx = 0; sidx < 32; ++sidx) {
                const float dr = __shfl_sync(0xffffffffu, d_raw, sidx);
                if (dr == 0.0f) continue;                        // warp-uniform
                float e[LF];
#pragma unroll
                for (int i = 0; i < LF; ++i) e[i] = __shfl_sync(0xffffffffu, enc[i], sidx);
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    float h = b0r[u];
#pragma unroll
                    for (int i = 0; i < LF; ++i) h = fmaf(w0r[u][i], e[i], h);
                    const bool on = h > 0.0f;
                    const float dh = on ? dr * w1r[u] : 0.0f;
#pragma unroll
                    for (int i = 0; i < LF; ++i) acc_w0[u][i] = fmaf(dh, e[i], acc_w0[u][i]);
                    acc_b0[u] += dh;
                    acc_w1[u] = fmaf(dr, on ? h : 0.0f, acc_w1[u]);
                }
            }
        }
    }
    // ---- flush: CTA sum in shared memory, one atomic per weight and CTA
#pragma unroll
    for (int u = 0; u < 2; ++u) {
        const int j = lane + 32 * u;
#pragma unroll
        for (int i = 0; i < LF; ++i) atomicAdd(&red[j * LF + i], acc_w0[u][i]);
        atomicAdd(&red[PL_HID * LF + j], acc_b0[u]);
        atomicAdd(&red[PL_HID * LF + PL_HID + j], acc_w1[u]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc_b1 += __shfl_xor_sync(0xffffffffu, acc_b1, o);
    if (lane == 0) atomicAdd(&red[PL_HID * LF + 2 * PL_HID], acc_b1);
    __syncthreads();
    for (int e = tid; e < PL_HID * LF + 2 * PL_HID + 1; e += PL_WARPS * 32) {
        const float v = red[e];
        float* dst = e < PL_HID * LF ? p.d_w0 + e
                   : e < PL_HID * LF + PL_HID ? p.d_b0 + (e - PL_HID * LF)
                   : e < PL_HID * LF + 2 * PL_HID ? p.d_w1 + (e - PL_HID * LF - PL_HID)
                   : p.d_b1;
        if (v != 0.0f) atomicAdd(dst, v);
    }
}

}  // namespace emer

using namespace emer;

extern "C" int emer_prop_level(const emer_grid_desc* g, const float* prev_s, const float* prev_cdf, int m1, int n,
                               const float* bias, float s_min, float s_max, int stot_kind, const float* origins,
                               const float* dirs, const float* aabb6, int unbounded, const float* table,
                               const float* w0, const float* b0, const float* w1, const float* b1, float* out_s,
                               float* out_t, float* out_cdf, float* out_sigma, int64_t n_rays, void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(g && prev_s && prev_cdf && origins && dirs && aabb6 && table && w0 && b0 && w1 && b1 && out_s &&
                     out_t && out_cdf,
                 "emer_prop_level: NULL pointer");
    EMER_REQUIRE(g->n_dims == 3, "emer_prop_level: proposal grids are 3-D");
    EMER_REQUIRE(g->n_levels * g->n_feat <= PL_MAX_IN && g->n_feat <= 4, "emer_prop_level: at most %d grid features",
                 PL_MAX_IN);
    EMER_REQUIRE(m1 >= 2 && n >= 1 && n + 1 <= PL_MAX_EDGES, "emer_prop_level: n=%d out of range", n);
    PropParams p;
    p.g = *g;
    p.prev_s = prev_s; p.prev_cdf = prev_cdf; p.bias = bias; p.origins = origins; p.dirs = dirs; p.aabb = aabb6;
    p.table = table; p.w0 = w0; p.b0 = b0; p.w1 = w1; p.b1 = b1; p.out_s = out_s; p.out_t = out_t; p.out_cdf = out_cdf;
    p.out_sigma = out_sigma;
    p.n_rays = n_rays; p.m1 = m1; p.n = n; p.stot_kind = stot_kind; p.unbounded = unbounded; p.s_min = s_min; p.s_max = s_max;
    const unsigned blocks = (unsigned)ceil_div(n_rays, PL_WARPS);
    cudaStream_t st = (cudaStream_t)stream;
    const int lf = g->n_levels * g->n_feat;
    if (g->n_feat == 1 && lf == 8) prop_level_kernel<8><<<blocks, PL_WARPS * 32, 0, st>>>(p);
    else if (g->n_feat == 1 && lf == 4) prop_level_kernel<4><<<blocks, PL_WARPS * 32, 0, st>>>(p);
    else prop_level_kernel<0><<<blocks, PL_WARPS * 32, 0, st>>>(p);
    return check_launch("emer_prop_level");
}

extern "C" int emer_prop_level_bwd(const emer_grid_desc* g, const float* t_edges, const float* sigma, const float* d_cdf,
                                   int n, const float* origins, const float* dirs, const float* aabb6, int unbounded,
                                   const float* table, const float* w0, const float* b0, const float* w1, float* xc,
                                   float* d_enc, float* d_w0, float* d_b0, float* d_w1, float* d_b1, int64_t n_rays,
                                   void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(g && t_edges && sigma && d_cdf && origins && dirs && aabb6 && table && w0 && b0 && w1 && xc && d_enc &&
                     d_w0 && d_b0 && d_w1 && d_b1,
                 "emer_prop_level_bwd: NULL pointer");
    const int lf = g->n_levels * g->n_feat;
    EMER_REQUIRE(g->n_dims == 3 && g->n_feat == 1 && (lf == 8 || lf == 4),
                 "emer_prop_level_bwd: 3-D grids of 4 or 8 levels x 1 feature (got %d levels x %d)", g->n_levels, g->n_feat);
    EMER_REQUIRE(n >= 1 && n + 1 <= PL_MAX_EDGES, "emer_prop_level_bwd: n=%d out of range", n);
    EMER_REQUIRE(((uintptr_t)d_enc & 15) == 0, "emer_prop_level_bwd: d_enc must be 16-byte aligned");
    PropBwdParams p;
    p.g = *g;
    p.t_edges = t_edges; p.sigma = sigma; p.d_cdf = d_cdf; p.origins = origins; p.dirs = dirs; p.aabb = aabb6;
    p.table = table; p.w0 = w0; p.b0 = b0; p.w1 = w1; p.xc = xc; p.d_enc = d_enc; p.d_w0 = d_w0; p.d_b0 = d_b0;
    p.d_w1 = d_w1; p.d_b1 = d_b1; p.n_rays = n_rays; p.n = n; p.unbounded = unbounded;
    int64_t blocks = ceil_div(n_rays, PL_WARPS);
    const int64_t resident = (int64_t)sm_count() * 3;            // persistent: the weight gradients flush once per CTA
    if (blocks > resident) blocks = resident;
    cudaStream_t st = (cudaStream_t)stream;
    if (lf == 8) prop_level_bwd_kernel<8><<<(unsigned)blocks, PL_WARPS * 32, 0, st>>>(p);
    else prop_level_bwd_kernel<4><<<(unsigned)blocks, PL_WARPS * 32, 0, st>>>(p);
    return check_launch("emer_prop_level_bwd");
}
