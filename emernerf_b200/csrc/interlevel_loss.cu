// Anti-aliased interlevel (proposal) loss of one proposal level, forward AND gradient, in one launch.
//
// Reference: PropNetEstimator.compute_loss, third_party/nerfacc_prop_net.py:182-240 with blur_stepfun (:22-34) and
// sorted_interp_quad (:37-60) -- per level ~40 torch launches (two sorts in the reference; two searchsorted + four
// scatters + three cumsums + six gathers in the drop-in's torch restatement) over [R, 2(S+1)] / [R, n+1] rows, and as
// many again in autograd's backward.  The loss reaches the proposal network only through the level's CDF row, the
// blurred target is a constant (detached), and everything is a per-ray computation on <= 260 numbers: one warp per ray,
// rows in shared memory.
//
//   y_j     = (cdf_{j+1} - cdf_j) / (s_{j+1} - s_j)                          final level, j < S          (:202-204)
//   knots   = merge(s - r, s + r)        (both halves sorted: rank = own index + lower/upper bound in the other half)
//   w       = [0, clamp_min(cumsum(diff(knots) * cumsum(+-slope)), 0)]       slope_j = (y_j - y_{j-1}) / 2r   (:22-34)
//   cdf_r   = [0, cumsum(0.5 (w_{i+1} + w_i) diff(knots))]                                               (:207-222)
//   q_k     = cdf_r[lo] + (x - knot_lo) (p_lo + p_hi f + p_lo (1 - f)) / 2   at x = prop_s_k             (:37-60)
//   term_k  = max(dq_k - dP_k, 0)^2 / (dP_k + 1e-5),  dP_k = prop_cdf_{k+1} - prop_cdf_k                 (:232-238)
//   out: sum_k term_k (accumulated into *loss_sum), d(sum term)/d prop_cdf -> d_prop_cdf [R, n+1]
// The caller divides by R n (the reference's .mean()) and applies the upstream gradient.
// The row is computed in fp64 from the fp32 inputs: dq_k is a difference of neighbouring values of a cumulative area
// that reaches ~1, and the hinge divides it by dP_k + 1e-5, so in fp32 the rounding of cdf_r alone (6e-8) put the
// gradient of a fine level (pulse width 0.003) 4e-3 off its fp64 value.
#include "common.cuh"

namespace emer {

constexpr int IL_WARPS = 4;
constexpr int IL_MAX_M = 129;              // final edges (S + 1)
constexpr int IL_MAX_K = 2 * IL_MAX_M;     // blurred knots
constexpr int IL_MAX_N1 = 257;             // proposal edges (n + 1)

struct InterlevelParams {
    const float* s;          // [R, m]   final-level edges (normalised distances)
    const float* cdf;        // [R, m]   final-level CDF (constant)
    const float* prop_s;     // [R, n1]
    const float* prop_cdf;   // [R, n1]
    float* loss_sum;         // [1] accumulated
    float* d_prop_cdf;       // [R, n1] or null
    int64_t n_rays;
    int m, n1;
    float r;
};

__global__ void __launch_bounds__(IL_WARPS * 32) interlevel_loss_kernel(const InterlevelParams p) {
    __shared__ double knot[IL_WARPS][IL_MAX_K + 2];
    __shared__ double wv[IL_WARPS][IL_MAX_K + 2];      // the blurred heights w
    __shared__ double cr[IL_WARPS][IL_MAX_K + 2];      // cdf of the blurred step function
    __shared__ double qv[IL_WARPS][IL_MAX_K + 2];       // merged +-slope jumps; later the interpolated cdf at the proposal edges
    static_assert(IL_MAX_K + 2 >= IL_MAX_N1, "qv holds both");
    __shared__ double blk[IL_WARPS];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int m = p.m, n1 = p.n1, K = 2 * m;
    const double r = p.r;
    double loss = 0.0;
    for (int64_t ray = (int64_t)blockIdx.x * IL_WARPS + wid; ray < p.n_rays; ray += (int64_t)gridDim.x * IL_WARPS) {
        const float* s = p.s + ray * m;
        const float* c = p.cdf + ray * m;
        __syncwarp();
        // ---- merge s - r and s + r; the slope jump of knot j travels with it
        for (int j = lane; j < m; j += 32) {
            const double sj = __ldg(s + j);
            const double a = sj - r, b = sj + r;
            const double y_hi = j < m - 1 ? ((double)__ldg(c + j + 1) - __ldg(c + j)) / (__ldg(s + j + 1) - sj) : 0.0;
            const double y_lo = j > 0 ? ((double)__ldg(c + j) - __ldg(c + j - 1)) / (sj - __ldg(s + j - 1)) : 0.0;
            const double slope = (y_hi - y_lo) / (2.0 * r);
            // rank of a_j: j + #{i: s_i + r < a_j};  rank of b_j: j + #{i: s_i - r <= b_j}
            int lo = 0, hi = m;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if ((double)__ldg(s + mid) + r < a) lo = mid + 1; else hi = mid;
            }
            const int ra = j + lo;
            lo = 0; hi = m;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if ((double)__ldg(s + mid) - r <= b) lo = mid + 1; else hi = mid;
            }
            const int rb = j + lo;
            knot[wid][ra] = a; qv[wid][ra] = slope;
            knot[wid][rb] = b; qv[wid][rb] = -slope;
        }
        __syncwarp();
        // ---- heights: w_0 = 0, w_{i+1} = max(cumsum_i((knot_{i+1} - knot_i) * cumsum_i(dslope)), 0); areas -> cdf_r
        double carry_s = 0.0, carry_h = 0.0, carry_a = 0.0, w_prev_last = 0.0;
        for (int i0 = 0; i0 < K - 1; i0 += 32) {
            const int i = i0 + lane;
            const bool ok = i < K - 1;
            const double ds = ok ? qv[wid][i] : 0.0;
            const double dk = ok ? knot[wid][i + 1] - knot[wid][i] : 0.0;
            const double cs = carry_s + warp_scan_incl(ds, lane);
            const double inc = dk * cs;
            const double hs = carry_h + warp_scan_incl(inc, lane);
            const double w_next = fmax(hs, 0.0);                               // w_{i+1}
            double w_cur = __shfl_up_sync(0xffffffffu, w_next, 1);             // w_i
            if (lane == 0) w_cur = w_prev_last;
            const double area = ok ? 0.5 * (w_next + w_cur) * dk : 0.0;
            const double ca = carry_a + warp_scan_incl(area, lane);
            if (ok) { wv[wid][i + 1] = w_next; cr[wid][i + 1] = ca; }
            carry_s = __shfl_sync(0xffffffffu, cs, 31);
            carry_h = __shfl_sync(0xffffffffu, hs, 31);
            carry_a = __shfl_sync(0xffffffffu, ca, 31);
            w_prev_last = __shfl_sync(0xffffffffu, w_next, 31);
        }
        if (lane == 0) { wv[wid][0] = 0.0; cr[wid][0] = 0.0; }
        __syncwarp();
        // ---- quadratic interpolation of cdf_r at the proposal edges
        const float* ps = p.prop_s + ray * n1;
        const float* pc = p.prop_cdf + ray * n1;
        for (int k = lane; k < n1; k += 32) {
            const double x = __ldg(ps + k);
            int lo = 0, hi = K;                                                // #{knots <= x}
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (knot[wid][mid] <= x) lo = mid + 1; else hi = mid;
            }
            const int i_lo = max(lo - 1, 0), i_hi = min(lo, K - 1);
            const double x_lo = knot[wid][i_lo], x_hi = knot[wid][i_hi];
            const double p_lo = wv[wid][i_lo], p_hi = wv[wid][i_hi];
            double f = (x - x_lo) / (x_hi - x_lo);
            if (f != f) f = 0.0;                                               // nan_to_num(., 0); +-inf clip below
            f = fmin(fmax(f, 0.0), 1.0);
            qv[wid][k] = cr[wid][i_lo] + (x - x_lo) * (p_lo + p_hi * f + p_lo * (1.0 - f)) / 2.0;
        }
        __syncwarp();
        // ---- terms and their derivative w.r.t. dP_k
        double g_prev_last = 0.0;                                              // g_{k0 - 1}
        for (int k0 = 0; k0 < n1; k0 += 32) {                                  // k = n1 - 1 only closes the gradient row
            const int k = k0 + lane;
            double g = 0.0;
            if (k < n1 - 1) {
                const double dq = qv[wid][k + 1] - qv[wid][k];
                const double dp = (double)__ldg(pc + k + 1) - __ldg(pc + k);
                const double d = fmax(dq - dp, 0.0);
                const double den = dp + 1e-5;
                loss += d * d / den;
                g = -2.0 * d / den - (d * d) / (den * den);
            }
            if (p.d_prop_cdf) {
                double g_prev = __shfl_up_sync(0xffffffffu, g, 1);
                if (lane == 0) g_prev = g_prev_last;
                if (k < n1) p.d_prop_cdf[ray * n1 + k] = (float)(g_prev - g);          // dP_{k-1} = P_k - P_{k-1}, dP_k = P_{k+1} - P_k
                g_prev_last = __shfl_sync(0xffffffffu, g, 31);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) loss += __shfl_xor_sync(0xffffffffu, loss, o);
    if (lane == 0) blk[wid] = loss;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < IL_WARPS; ++w) t += blk[w];
        if (t != 0.0) atomicAdd(p.loss_sum, (float)t);
    }
}

}  // namespace emer

using namespace emer;

extern "C" int emer_interlevel_loss(const float* s, const float* cdf, int m, const float* prop_s, const float* prop_cdf,
                                    int n1, float pulse_width, float* loss_sum, float* d_prop_cdf, int64_t n_rays,
                                    void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(s && cdf && prop_s && prop_cdf && loss_sum, "emer_interlevel_loss: NULL pointer");
    EMER_REQUIRE(m >= 2 && m <= IL_MAX_M && n1 >= 2 && n1 <= IL_MAX_N1,
                 "emer_interlevel_loss: %d final edges / %d proposal edges out of range (<= %d / <= %d)", m, n1, IL_MAX_M,
                 IL_MAX_N1);
    EMER_REQUIRE(pulse_width > 0.0f, "emer_interlevel_loss: pulse width must be positive");
    InterlevelParams p{s, cdf, prop_s, prop_cdf, loss_sum, d_prop_cdf, n_rays, m, n1, pulse_width};
    int64_t blocks = ceil_div(n_rays, IL_WARPS);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    interlevel_loss_kernel<<<(unsigned)blocks, IL_WARPS * 32, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_interlevel_loss");
}
