// Scene contraction + in-cube selector of one point, for every kernel that feeds a hash grid (elementwise.cu,
// prop_level.cu).  Reference: radiance_fields/nerf_utils.py:13-28,59-75.
#pragma once
#include "common.cuh"

namespace emer {

// aabb[6] = (lo, hi)
__device__ __forceinline__ void load_box(const float* __restrict__ aabb, float (&lo)[3], float (&hi)[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) { lo[d] = __ldg(aabb + d); hi[d] = __ldg(aabb + 3 + d); }
}

// Forward arithmetic in exactly the reference's operation order (no FMA contraction):
//   xn = (x - lo) / (hi - lo) * 2 - 1 ; mag = max_i |xn_i|
//   y  = mag < 1 ? xn : (2 - 1/mag) * (xn / mag) ; out = y / 4 + 0.5 ; out *= all(0 < out < 1)
// lo / hi: the box (load_box).  xn, mag, amax (the arg-max coordinate) and sel are what the backward needs.
__device__ __forceinline__ void contract_point(const float (&x)[3], const float (&lo)[3], const float (&hi)[3],
                                               int unbounded, int apply_selector, float (&out)[3],
                                               float (&xn)[3], float& mag, int& amax, bool& sel) {
    float m = -1.0f;
    int am = 0;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float t = (x[d] - lo[d]) / (hi[d] - lo[d]);
        if (unbounded) t = t * 2.0f - 1.0f;
        xn[d] = t;
        float a = fabsf(t);
        if (a > m) { m = a; am = d; }
    }
    mag = m;
    amax = am;
    bool s = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float y;
        if (unbounded) {
            y = (m < 1.0f) ? xn[d] : (2.0f - 1.0f / m) * (xn[d] / m);
            y = y / 4.0f + 0.5f;
        } else {
            y = xn[d];
        }
        out[d] = y;
        s = s && (y > 0.0f) && (y < 1.0f);
    }
    if (!apply_selector) s = true;
    sel = s;
    if (!s) {
#pragma unroll
        for (int d = 0; d < 3; ++d) out[d] = out[d] * 0.0f;   // keeps NaN propagation of `p * selector`
    }
}

}  // namespace emer
