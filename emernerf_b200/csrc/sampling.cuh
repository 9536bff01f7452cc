// The s->t warp and one output edge of the inverse-CDF resampling, for every kernel that draws sample positions
// (sampling.cu, prop_level.cu): one body, so every kind of step draws bit-identical edges from identical CDF rows.
// fp32, operation by operation in the order of nerfacc.pdf.importance_sampling and _transform_stot
// (third_party/nerfacc_prop_net.py:153,172 and :317-339 of the reference).
#pragma once
#include "common.cuh"

namespace emer {

__device__ __forceinline__ float s_to_t(float s, float s_min, float s_max, int kind) {
    // icontract(s * s_max + (1 - s) * s_min)
    const float v = s * s_max + (1.0f - s) * s_min;
    switch (kind) {
        case EMER_STOT_UNIFORM: return v;
        case EMER_STOT_LINDISP: return 1.0f / v;
        case EMER_STOT_SQRT: return v * v;
        case EMER_STOT_LOG: return expf(v);
        // torch evaluates `200 / x` as reciprocal(x) * 200 (Tensor.__rtruediv__): two roundings
        case EMER_STOT_UNIFORM_LINDISP: return v < 0.5f ? v * 400.0f : (1.0f / (2.0f - 2.0f * v)) * 200.0f;
        default: return v < 0.5f ? 2.0f * v : 1.0f / (2.0f - 2.0f * v);
    }
}

// Edge k of the n intervals resampled from one ray's CDF row c over the edges v (m1 entries each); bias is the ray's
// jitter (0.5 when not stratified).  Returns s; bin is the upper bound of u in c, in [0, m1].
__device__ __forceinline__ float resample_edge(const float* __restrict__ c, const float* __restrict__ v, int m1, int n,
                                               int k, float bias, int& bin) {
    const float u_floor = __ldg(c);
    const float u_ceil = __ldg(c + m1 - 1);
    const float u_step = (u_ceil - u_floor) / (float)n;
    const float u = u_floor + ((float)k + (bias - 0.5f)) * u_step;
    // upper bound: first p in [0, m1] with c[p] > u
    int lo = 0, hi = m1;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(c + mid) > u) hi = mid;
        else lo = mid + 1;
    }
    bin = lo;
    const int p0 = min(max(lo - 1, 0), m1 - 1);
    const int p1 = min(max(lo, 0), m1 - 1);
    const float u_lo = __ldg(c + p0), u_hi = __ldg(c + p1);
    const float t_lo = __ldg(v + p0), t_hi = __ldg(v + p1);
    const float du = u_hi - u_lo;
    if (du < 1e-10f) return (t_lo + t_hi) * 0.5f;
    return (u - u_lo) * ((t_hi - t_lo) / du) + t_lo;
}

}  // namespace emer
