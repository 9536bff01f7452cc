// Point-wise pieces of the path: scene contraction (+selector, +time column) and the
// trunc_exp density activation.  HBM-bound streaming kernels: 24-32 B/point (contract),
// 8 B/point (trunc_exp).  Reference: radiance_fields/nerf_utils.py:13-28,59-75;
// radiance_fields/radiance_field.py:278-300,828-835.
#include "common.cuh"
#include "contract.cuh"

namespace emer {

__global__ void contract_fwd_kernel(const float* __restrict__ pos, const float* __restrict__ aabb,
                                    const float* __restrict__ time, float* __restrict__ out,
                                    int out_dim, int unbounded, int apply_selector, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x[3] = {__ldg(pos + i * 3), __ldg(pos + i * 3 + 1), __ldg(pos + i * 3 + 2)};
    float lo[3], hi[3], o[3], xn[3], mag;
    int am;
    bool sel;
    load_box(aabb, lo, hi);
    contract_point(x, lo, hi, unbounded, apply_selector, o, xn, mag, am, sel);
    if (out_dim == 4) {
        reinterpret_cast<float4*>(out)[i] = make_float4(o[0], o[1], o[2], time ? __ldg(time + i) : 0.0f);
    } else {
        out[i * 3] = o[0];
        out[i * 3 + 1] = o[1];
        out[i * 3 + 2] = o[2];
    }
}

__global__ void contract_bwd_kernel(const float* __restrict__ pos, const float* __restrict__ aabb,
                                    const float* __restrict__ dout, float* __restrict__ dpos,
                                    float* __restrict__ dtime, int out_dim, int unbounded, int apply_selector,
                                    int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x[3] = {__ldg(pos + i * 3), __ldg(pos + i * 3 + 1), __ldg(pos + i * 3 + 2)};
    float lo[3], hi[3], o[3], xn[3], mag;
    int am;
    bool sel;
    load_box(aabb, lo, hi);
    contract_point(x, lo, hi, unbounded, apply_selector, o, xn, mag, am, sel);
    float g[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) g[d] = sel ? __ldg(dout + i * out_dim + d) : 0.0f;
    if (dtime && out_dim == 4) dtime[i] = __ldg(dout + i * 4 + 3);
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
            const float sgn = xn[am] > 0.0f ? 1.0f : (xn[am] < 0.0f ? -1.0f : 0.0f);
            const float extra = dot * (2.0f * inv - 2.0f) * inv * inv * sgn;
#pragma unroll
            for (int d = 0; d < 3; ++d)
                if (d == am) gxn[d] += extra;
        }
    } else {
#pragma unroll
        for (int d = 0; d < 3; ++d) gxn[d] = g[d];
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float k = (unbounded ? 2.0f : 1.0f) / (hi[d] - lo[d]);
        dpos[i * 3 + d] = gxn[d] * k;
    }
}

__global__ void trunc_exp_fwd_kernel(const float* __restrict__ x, int64_t ldx, float* __restrict__ y,
                                     int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) y[i] = density_fwd(__ldg(x + i * ldx));
}

__global__ void trunc_exp_bwd_kernel(const float* __restrict__ x, int64_t ldx,
                                     const float* __restrict__ dy, float* __restrict__ dx, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) dx[i] = density_bwd(__ldg(dy + i), __ldg(x + i * ldx));
}

}  // namespace emer

using namespace emer;

extern "C" int emer_contract_fwd(const float* pos, const float* aabb6, const float* time, float* out,
                                 int out_dim, int unbounded, int apply_selector, int64_t n, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(pos && aabb6 && out, "emer_contract_fwd: NULL pointer");
    EMER_REQUIRE(out_dim == 3 || out_dim == 4, "emer_contract_fwd: out_dim must be 3 or 4");
    EMER_REQUIRE(out_dim == 3 || ((uintptr_t)out & 15) == 0, "emer_contract_fwd: out must be 16-byte aligned");
    contract_fwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(pos, aabb6, time, out, out_dim,
                                                                                      unbounded, apply_selector, n);
    return check_launch("emer_contract_fwd");
}

extern "C" int emer_contract_bwd(const float* pos, const float* aabb6, const float* dout, float* dpos,
                                 float* dtime, int out_dim, int unbounded, int apply_selector, int64_t n,
                                 void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(pos && aabb6 && dout && dpos, "emer_contract_bwd: NULL pointer");
    EMER_REQUIRE(out_dim == 3 || out_dim == 4, "emer_contract_bwd: out_dim must be 3 or 4");
    contract_bwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(pos, aabb6, dout, dpos, dtime,
                                                                                      out_dim, unbounded, apply_selector, n);
    return check_launch("emer_contract_bwd");
}

extern "C" int emer_trunc_exp_fwd(const float* x, int64_t ldx, float* y, int64_t n, void* stream) {
    if (n == 0) return 0;
    trunc_exp_fwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, ldx, y, n);
    return check_launch("emer_trunc_exp_fwd");
}

extern "C" int emer_trunc_exp_bwd(const float* x, int64_t ldx, const float* dy, float* dx, int64_t n,
                                  void* stream) {
    if (n == 0) return 0;
    trunc_exp_bwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, ldx, dy, dx, n);
    return check_launch("emer_trunc_exp_bwd");
}
