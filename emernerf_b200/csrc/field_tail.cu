// "Field tail": everything between the base MLP and the colour head, in one launch each way.
//
// Reference (radiance_fields/radiance_field.py:417-422,622-647): split geo features, density =
// trunc_exp(geo[..., 0] - 1), directions -> (d+1)/2 -> sinusoidal encoding (33), appearance embedding
// gather (16), torch.cat([h, emb, geo]) -> rgb head.  In torch that is ~12 launches and three
// [N, 113]-sized copies per call (plus a sort-based embedding backward).  Here:
//
//   forward : rgb_in[n, 0:64] = feats[n, 0:G]            (geo first: 16-byte aligned gradient view)
//             rgb_in[n, G:G+33] = sinenc((dir[ray]+1)/2)  rgb_in[n, G+33:G+33+E] = emb[idx[ray]]
//             rgb_in[n, pad] = 0                          sigma[n] = exp(feats[n, 0] - 1)
//   backward: d_feats = d_rgb_in[:, 0:G] (a view, nothing copied) with column 0 += d_sigma * exp(clamp)
//             d_emb[idx[ray]] += sum_s d_rgb_in[ray, s, emb columns]       (warp reduce + 16 atomics)
//
// The rgb head's weight columns are permuted to this [geo | dir | emb] order by the caller.
// HBM-bound: (G + ld_out)*4 B/point forward.
#include "common.cuh"

namespace emer {

constexpr int FT_DIR = 33;   // 3 identity + 5 octaves x (sin, sin(.+pi/2)) x 3

// One CTA per ray: the per-ray tail (direction encoding + embedding row, <= 64 floats) is computed once
// into shared memory, then the ray's S rows are written as 16-byte pieces: geo columns are a straight
// float4 copy of the field features, tail columns a broadcast of the shared values.
constexpr int FT_MAX_TAIL = 72;      // 33 + E (<= 32) + pad

__global__ void __launch_bounds__(256) field_tail_fwd_kernel(const float* __restrict__ feats, int64_t ld_feats, int G,
                                                              const float* __restrict__ dirs,
                                                              const int64_t* __restrict__ idx,
                                                              const float* __restrict__ emb, int E,
                                                              float* __restrict__ out, int64_t ld_out, int out_cols,
                                                              float* __restrict__ sigma, int64_t n_rays, int S) {
    __shared__ __align__(16) float tail[FT_MAX_TAIL];
    const int64_t ray = blockIdx.x;
    const int tid = threadIdx.x;
    const int n_tail = out_cols - G;                         // includes the zero padding
    if (tid < n_tail) {
        float x = 0.0f;
        if (tid < FT_DIR) {
            const int e = tid;                                // [x(3) | sin(2^i x)(15) | sin(2^i x + pi/2)(15)]
            if (e < 3) {
                x = (__ldg(dirs + ray * 3 + e) + 1.0f) / 2.0f;
            } else {
                const int q = (e - 3) % 15, shifted = (e - 3) / 15;
                const int oct = q / 3, d = q % 3;
                const float u = (__ldg(dirs + ray * 3 + d) + 1.0f) / 2.0f;
                float arg = u * (float)(1 << oct);
                if (shifted) arg = arg + 0.5f * 3.14159265358979323846f;
                x = sinf(arg);
            }
        } else if (tid < FT_DIR + E) {
            x = __ldg(emb + __ldg(idx + ray) * E + (tid - FT_DIR));
        }
        tail[tid] = x;
    }
    __syncthreads();
    const int quads = out_cols / 4, gq = G / 4;
    const bool vec_in = (ld_feats % 4 == 0) && ((reinterpret_cast<uintptr_t>(feats) & 15) == 0);
    for (int e = tid; e < S * quads; e += 256) {
        const int s = e / quads, q = e - s * quads;
        const int64_t pt = ray * S + s;
        float4 v;
        if (q < gq) {
            const float* src = feats + pt * ld_feats + q * 4;
            if (vec_in) v = __ldg(reinterpret_cast<const float4*>(src));
            else v = make_float4(__ldg(src), __ldg(src + 1), __ldg(src + 2), __ldg(src + 3));
            if (q == 0 && sigma) sigma[pt] = density_fwd(v.x);
        } else {
            v = *reinterpret_cast<const float4*>(tail + (q - gq) * 4);
        }
        *reinterpret_cast<float4*>(out + pt * ld_out + q * 4) = v;
    }
}

// d_rgb_in[:, 0] += d_sigma * exp(min(feats0 - 1, 15)); d_emb scatter.  One warp per ray.
__global__ void __launch_bounds__(256) field_tail_bwd_kernel(const float* __restrict__ feats, int64_t ld_feats,
                                                              float* __restrict__ d_out, int64_t ld_out, int G,
                                                              const float* __restrict__ d_sigma,
                                                              const int64_t* __restrict__ idx, float* __restrict__ d_emb,
                                                              int E, int64_t n_rays, int S) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    if (ray >= n_rays) return;
    if (d_sigma) {
        for (int s = lane; s < S; s += 32) {
            const int64_t pt = ray * S + s;
            const float g = __ldg(d_sigma + pt);
            if (g != 0.0f) d_out[pt * ld_out] += density_bwd(g, __ldg(feats + pt * ld_feats));
        }
    }
    if (d_emb) {
        // lanes 0..E-1 own one embedding column each (E <= 32)
        float acc = 0.0f;
        if (lane < E) {
            const float* p = d_out + ray * S * ld_out + G + FT_DIR + lane;
            for (int s = 0; s < S; ++s) acc += p[(int64_t)s * ld_out];
            atomicAdd(d_emb + __ldg(idx + ray) * E + lane, acc);
        }
    }
}

}  // namespace emer

using namespace emer;

extern "C" int emer_field_tail_fwd(const float* feats, int64_t ld_feats, int g_dim, const float* dirs,
                                   const int64_t* idx, const float* emb, int e_dim, float* out, int64_t ld_out,
                                   float* sigma, int64_t n_rays, int n_samples, void* stream) {
    if (n_rays == 0) return 0;
    EMER_REQUIRE(feats && dirs && out, "emer_field_tail_fwd: NULL pointer");
    EMER_REQUIRE(e_dim == 0 || (idx && emb), "emer_field_tail_fwd: embedding needs indices and a table");
    EMER_REQUIRE(ld_out % 4 == 0 && ld_out >= g_dim + FT_DIR + e_dim && ((uintptr_t)out & 15) == 0,
                 "emer_field_tail_fwd: output rows must be 16-byte aligned and wide enough");
    // columns [0, out_cols) of every row are written (the padding with zeros); ld_out is only the row stride,
    // so the rows may live inside a wider buffer (the rgb head's skip-concatenation buffer)
    const int out_cols = (g_dim + FT_DIR + e_dim + 3) / 4 * 4;
    EMER_REQUIRE(g_dim % 4 == 0 && out_cols - g_dim <= FT_MAX_TAIL, "emer_field_tail_fwd: geometry width %d must be a "
                 "multiple of 4 and the tail at most %d floats", g_dim, FT_MAX_TAIL);
    field_tail_fwd_kernel<<<(unsigned)n_rays, 256, 0, (cudaStream_t)stream>>>(
        feats, ld_feats, g_dim, dirs, idx, emb, e_dim, out, ld_out, out_cols, sigma, n_rays, n_samples);
    return check_launch("emer_field_tail_fwd");
}

extern "C" int emer_field_tail_bwd(const float* feats, int64_t ld_feats, float* d_out, int64_t ld_out, int g_dim,
                                   const float* d_sigma, const int64_t* idx, float* d_emb, int e_dim, int64_t n_rays,
                                   int n_samples, void* stream) {
    if (n_rays == 0 || (!d_sigma && !d_emb)) return 0;
    EMER_REQUIRE(feats && d_out, "emer_field_tail_bwd: NULL pointer");
    EMER_REQUIRE(e_dim <= 32, "emer_field_tail_bwd: embedding width %d > 32", e_dim);
    field_tail_bwd_kernel<<<(unsigned)ceil_div(n_rays, 8), 256, 0, (cudaStream_t)stream>>>(
        feats, ld_feats, d_out, ld_out, g_dim, d_sigma, idx, d_emb, e_dim, n_rays, n_samples);
    return check_launch("emer_field_tail_bwd");
}
