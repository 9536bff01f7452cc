// Inverse-CDF resampling of ray intervals + the s->t warp.
//
// Replaces nerfacc.pdf.importance_sampling (the one nerfacc CUDA kernel the reference hits by
// default, third_party/nerfacc_prop_net.py:153,172) and _transform_stot (:317-339).
// Integer work (upper-bound bin per output edge) is bit-exact against the oracle; the fp32
// arithmetic (sampling.cuh, which the fused proposal level includes too) is written operation by
// operation in the oracle's order (library built with -fmad=false), so the produced s/t edges are
// bit-identical for identical CDFs.
//
// Layout: vals, cdfs [R, m1] row-major; outputs [R, n+1].  One thread per output edge;
// a ray's CDF row (<= 129 floats) is read through L1.  HBM-bound and tiny:
// (2*m1 + 2*(n+1)) * 4 bytes per ray.
#include "sampling.cuh"

namespace emer {

__global__ void pdf_resample_kernel(const float* __restrict__ vals, const float* __restrict__ cdfs,
                                    int m1, int n, const float* __restrict__ bias, float s_min,
                                    float s_max, int kind, float* __restrict__ out_s,
                                    float* __restrict__ out_t, int32_t* __restrict__ out_bins,
                                    int64_t total) {
    const int64_t tid = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= total) return;
    const int64_t ray = tid / (n + 1);
    const int k = (int)(tid - ray * (n + 1));
    int p;
    const float s = resample_edge(cdfs + ray * m1, vals + ray * m1, m1, n, k, bias ? __ldg(bias + ray) : 0.5f, p);
    out_s[tid] = s;
    if (out_t) out_t[tid] = s_to_t(s, s_min, s_max, kind);
    if (out_bins) out_bins[tid] = p;
}

}  // namespace emer

using namespace emer;

extern "C" int emer_pdf_resample(const float* vals, const float* cdfs, int m1, int n, const float* bias,
                                 float s_min, float s_max, int stot_kind, float* out_s, float* out_t,
                                 int32_t* out_bins, int64_t n_rays, void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(vals && cdfs && out_s, "emer_pdf_resample: NULL pointer");
    EMER_REQUIRE(m1 >= 2 && n >= 1, "emer_pdf_resample: need m1 >= 2 edges and n >= 1 intervals");
    EMER_REQUIRE(stot_kind >= 0 && stot_kind <= EMER_STOT_UNIFORM_LINDISP_0, "emer_pdf_resample: unknown s->t kind %d",
                 stot_kind);
    const int64_t total = n_rays * (n + 1);
    pdf_resample_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
        vals, cdfs, m1, n, bias, s_min, s_max, stot_kind, out_s, out_t, out_bins, total);
    return check_launch("emer_pdf_resample");
}
