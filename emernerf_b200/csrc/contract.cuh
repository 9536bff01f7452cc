// Scene contraction + in-cube selector of one point and its backward, for every kernel that feeds a hash grid
// (elementwise.cu, prop_level.cu, flow_branch.cu).  Reference: radiance_fields/nerf_utils.py:13-28,59-75.
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

// Backward of contract_point: dpos = J^T g for the output gradient g (the selector already applied, i.e. g = 0 where
// sel is false), from the xn / mag / amax the forward returned.
__device__ __forceinline__ void contract_point_bwd(const float (&g_in)[3], const float (&xn)[3], float mag, int amax,
                                                   const float (&lo)[3], const float (&hi)[3], int unbounded,
                                                   float (&dpos)[3]) {
    float g[3] = {g_in[0], g_in[1], g_in[2]};
    float gxn[3];
    if (unbounded) {
#pragma unroll
        for (int d = 0; d < 3; ++d) g[d] *= 0.25f;
        if (mag < 1.0f) {
#pragma unroll
            for (int d = 0; d < 3; ++d) gxn[d] = g[d];
        } else {
            const float inv = 1.0f / mag;
            const float u = 2.0f - inv;
            float dot = 0.0f;
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                gxn[d] = u * inv * g[d];
                dot = fmaf(g[d], xn[d], dot);
            }
            // d/dmag of (2 - 1/mag) * xn/mag, routed to the arg-max coordinate (inf-norm subgradient)
            const float sgn = xn[amax] > 0.0f ? 1.0f : (xn[amax] < 0.0f ? -1.0f : 0.0f);
            const float extra = dot * (2.0f * inv - 2.0f) * inv * inv * sgn;
#pragma unroll
            for (int d = 0; d < 3; ++d)
                if (d == amax) gxn[d] += extra;
        }
    } else {
#pragma unroll
        for (int d = 0; d < 3; ++d) gxn[d] = g[d];
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float k = (unbounded ? 2.0f : 1.0f) / (hi[d] - lo[d]);
        dpos[d] = gxn[d] * k;
    }
}

}  // namespace emer
