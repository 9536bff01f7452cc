// The flow warp of the flow variants' temporal aggregation, both directions in one launch each way.  Reference:
// radiance_fields/radiance_field.py:449-452 (temporal_aggregation):
//     w_pos  = contract_points(positions + flow * noise)            flow = forward_flow | backward_flow
//     w_time = clamp(t + sign * time_diff * noise, 0, 1)            sign = +1 | -1
// Row i of the output is the forward warp of point i, row n + i its backward warp: [x y z t] grid coordinates that the
// dynamic and flow grids read as one [2n, 4] block.  The backward takes those rows' input gradient (grid dx, the first
// three columns) to d_flow through the contraction's Jacobian, the selector and noise; time and noise carry no gradient.
#include "common.cuh"
#include "contract.cuh"

namespace emer {

// the warped point of row i in direction dir (0 forward, 1 backward), in torch's operation order (no contraction)
__device__ __forceinline__ void warp_point(const float* __restrict__ pos, const float* __restrict__ flow, float nz,
                                           int64_t i, int dir, float (&x)[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) x[d] = __fadd_rn(__ldg(pos + i * 3 + d), __fmul_rn(__ldg(flow + i * 6 + 3 * dir + d), nz));
}

__global__ void flow_warp_fwd_kernel(const float* __restrict__ pos, const float* __restrict__ flow,
                                     const float* __restrict__ noise, int64_t ld_noise, const float* __restrict__ t,
                                     const float* __restrict__ aabb, const float* __restrict__ time_diff, int unbounded,
                                     float* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float nz = noise ? __ldg(noise + i * ld_noise) : 1.0f;
    const float ti = __ldg(t + i), dt = __ldg(time_diff);
    float lo[3], hi[3];
    load_box(aabb, lo, hi);
#pragma unroll
    for (int dir = 0; dir < 2; ++dir) {
        float x[3], o[3], xn[3], mag;
        int am;
        bool sel;
        warp_point(pos, flow, nz, i, dir, x);
        contract_point(x, lo, hi, unbounded, 1, o, xn, mag, am, sel);
        float tw = __fadd_rn(ti, __fmul_rn(dir ? -dt : dt, nz));
        tw = tw < 0.0f ? 0.0f : (tw > 1.0f ? 1.0f : tw);          // torch.clamp: NaN stays NaN
        reinterpret_cast<float4*>(out)[dir * n + i] = make_float4(o[0], o[1], o[2], tw);
    }
}

__global__ void flow_warp_bwd_kernel(const float* __restrict__ pos, const float* __restrict__ flow,
                                     const float* __restrict__ noise, int64_t ld_noise, const float* __restrict__ aabb,
                                     int unbounded, const float* __restrict__ d_coords, float* __restrict__ d_flow,
                                     int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float nz = noise ? __ldg(noise + i * ld_noise) : 1.0f;
    float lo[3], hi[3];
    load_box(aabb, lo, hi);
#pragma unroll
    for (int dir = 0; dir < 2; ++dir) {
        float x[3], o[3], xn[3], mag, g[3], dp[3];
        int am;
        bool sel;
        warp_point(pos, flow, nz, i, dir, x);
        contract_point(x, lo, hi, unbounded, 1, o, xn, mag, am, sel);
        const float4 gc = __ldg(reinterpret_cast<const float4*>(d_coords) + dir * n + i);
        g[0] = sel ? gc.x : 0.0f;
        g[1] = sel ? gc.y : 0.0f;
        g[2] = sel ? gc.z : 0.0f;
        contract_point_bwd(g, xn, mag, am, lo, hi, unbounded, dp);
#pragma unroll
        for (int d = 0; d < 3; ++d) d_flow[i * 6 + 3 * dir + d] = __fmul_rn(dp[d], nz);
    }
}

}  // namespace emer

using namespace emer;

extern "C" int emer_flow_warp_fwd(const float* pos, const float* flow, const float* noise, int64_t ld_noise,
                                  const float* t, const float* aabb6, const float* time_diff, int unbounded, float* coords,
                                  int64_t n, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(pos && flow && t && aabb6 && time_diff && coords, "emer_flow_warp_fwd: NULL pointer");
    EMER_REQUIRE(((uintptr_t)coords & 15) == 0, "emer_flow_warp_fwd: coords must be 16-byte aligned");
    flow_warp_fwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(pos, flow, noise, ld_noise, t, aabb6,
                                                                                       time_diff, unbounded, coords, n);
    return check_launch("emer_flow_warp_fwd");
}

extern "C" int emer_flow_warp_bwd(const float* pos, const float* flow, const float* noise, int64_t ld_noise,
                                  const float* aabb6, int unbounded, const float* d_coords, float* d_flow, int64_t n,
                                  void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(pos && flow && aabb6 && d_coords && d_flow, "emer_flow_warp_bwd: NULL pointer");
    EMER_REQUIRE(((uintptr_t)d_coords & 15) == 0, "emer_flow_warp_bwd: d_coords must be 16-byte aligned");
    flow_warp_bwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(pos, flow, noise, ld_noise, aabb6,
                                                                                       unbounded, d_coords, d_flow, n);
    return check_launch("emer_flow_warp_bwd");
}
