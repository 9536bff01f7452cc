// The transmittance scan along one ray, shared by composite_fwd_kernel (composite.cu) and render_fwd_kernel
// (render.cu), so that the weights / trans / opacity / depth / median depth both kernels write are the same device
// code and therefore bit-identical.
//
// One warp per ray, lanes stride the samples: step() consumes one 32-sample chunk (this lane's sample s0 + lane),
// carrying the running sums of sigma*delta and of the weights between chunks; finish() reduces the ray totals.
#pragma once
#include "common.cuh"

namespace emer {

template <bool MEDIAN>
struct RayScan {
    float carry_e = 0.0f;     // sum of sigma*delta before this chunk
    float carry_w = 0.0f;     // sum of weights before this chunk
    float sum_w = 0.0f, sum_wm = 0.0f;
    float med = 0.0f;
    bool med_found = false;
    float last_mid = 0.0f;

    // weight of this lane's sample (0 when !ok); T receives its transmittance
    __device__ __forceinline__ float step(float a, float b, float sg, bool ok, int s0, int S, int lane, float& T) {
        const float x = ok ? sg * (b - a) : 0.0f;
        const float incl = warp_scan_incl(x, lane);
        const float e_excl = carry_e + (incl - x);
        T = expf(-e_excl);
        const float alpha = 1.0f - expf(-x);
        const float w = ok ? T * alpha : 0.0f;
        const float mid = (a + b) / 2.0f;
        if (MEDIAN) {
            const float w_incl = warp_scan_incl(w, lane);
            const float cw = carry_w + w_incl;
            // median: first sample with cumulative weight >= 0.5 (searchsorted side="left")
            const unsigned hit = __ballot_sync(0xffffffffu, ok && (cw >= 0.5f));
            if (!med_found && hit) {
                const int first = __ffs(hit) - 1;
                med = __shfl_sync(0xffffffffu, mid, first);
                med_found = true;
            }
            // last valid midpoint (index clamp to S-1 when the ray never reaches 0.5)
            const int last_lane = min(31, S - 1 - s0);
            last_mid = __shfl_sync(0xffffffffu, mid, last_lane);
            carry_w += __shfl_sync(0xffffffffu, w_incl, 31);
        }
        sum_w += w;
        sum_wm = fmaf(w, mid, sum_wm);
        carry_e += __shfl_sync(0xffffffffu, incl, 31);
        return w;
    }

    // on every lane after the last chunk: opacity clamped to [1e-6, 1], depth = sum w*mid / opacity, median depth
    __device__ __forceinline__ void finish(float& op, float& depth, float& median) {
        const float sw = warp_sum(sum_w);
        const float swm = warp_sum(sum_wm);
        op = fminf(fmaxf(sw, 1e-6f), 1.0f);
        depth = swm / op;
        median = med_found ? med : last_mid;
    }
};

}  // namespace emer
