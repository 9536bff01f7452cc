// The fused field chain on Hopper warpgroup MMA: hash-grid features -> base MLP -> density + colour head, ONE persistent
// kernel, activations never leave the registers.
//
// Replaces, for one [N, k_enc] block of hash-grid features (reference: radiance_fields/radiance_field.py)
//     feats = base_mlp(enc)                       Linear(k_enc,64)-ReLU-Linear(64, 64 [+64 semantic])     :74-80,314-318
//     sigma = trunc_exp(feats[:, 0] - 1)                                                                  :422
//     rgb   = sigmoid(rgb_head([dir enc | embedding | geo]))   MLP 113->64, [64|113]->64, 64->3, skip 1  :131-143,622-658
// which the per-layer path runs as 6 launches with every [N, 64..180] activation round-tripping HBM.
//
// Per-ray columns.  The colour head's input is [dir encoding (33) | appearance embedding (16) | geo (64)]; the first 49
// columns are the same for all samples of a ray, so  W[:, ray cols] * v_ray  is a per-RAY bias, computed once per ray
// by the caller (ray_bias[R, 128] = [b0 + W0[:, :49] v | b1 + W1[:, 64:113] v]).  The wide layers become
//     h0 = relu(geo W0g^T + ray_bias0[ray])            64 -> 64
//     h1 = relu(h0 W1h^T + geo W1g^T + ray_bias1[ray]) 128 -> 64
// and the [N, 113] / [N, 177] concatenations of the reference never exist.
//
// Tensor-core mapping (3xTF32, tc_common.cuh; DESIGN.md §5.1): each warpgroup walks its own 64-point tiles through all
// five layers; the weights are resident in shared memory, and the accumulator of layer i is the A operand of layer i+1.
#include "common.cuh"
#include "tc_common.cuh"

namespace emer {
namespace ff {

using namespace emer::tc;

constexpr int ROWS = 64;                      // points per tile = M of one wgmma
constexpr int WGS = 3;                        // warpgroups per CTA, each on its own tiles
constexpr int THREADS = WGS * 128;
constexpr int H = 64;                         // hidden / geometry / head width this kernel is specialised for

struct FwdParams {
    const float* enc; int64_t ld_enc; int k_enc;                  // [N, k_enc], k_enc % 8 == 0, <= 64
    const float *wb0, *bb0, *wb1, *bb1; int n_feat;               // base MLP; n_feat = 64 (geo) or 128 (geo | semantic)
    const float* w0g; int64_t ld_w0;                              // colour head layer 0, geo columns   [64, 64]
    const float *w1h, *w1g; int64_t ld_w1;                        // layer 1: hidden columns, geo columns [64, 64] each
    const float *w2, *b2;                                         // [3, 64], [3]
    const float* ray_bias; int samples;                           // [R, 128]; ray of point i = i / samples
    float *sigma, *rgb;                                           // [N], [N, 3]
    float *save_hb, *save_hg, *save_h1, *save_sem;                // training saves: [N,64], [N,128]=[h0|geo], [N,64], [N,64]
    int64_t n;
};

// shared-memory map (bytes): B operands as K-major panels (tc::b_off), hi and lo
struct Smem {
    int wb0_hi, wb0_lo, wb1_hi, wb1_lo, wg_hi, wg_lo, w1h_hi, w1h_lo, w2_hi, w2_lo, bias, total;
};
__host__ __device__ inline Smem smem_map(int k_enc, int n_feat) {
    Smem m;
    int o = 0;
    const int wb0 = (k_enc / 4) * H * 16, wb1 = (H / 4) * n_feat * 16, wg = (H / 4) * 128 * 16, w1h = (H / 4) * H * 16,
              w2 = (H / 4) * 8 * 16;
    m.wb0_hi = o; o += wb0; m.wb0_lo = o; o += wb0;
    m.wb1_hi = o; o += wb1; m.wb1_lo = o; o += wb1;
    m.wg_hi = o; o += wg; m.wg_lo = o; o += wg;
    m.w1h_hi = o; o += w1h; m.w1h_lo = o; o += w1h;
    m.w2_hi = o; o += w2; m.w2_lo = o; o += w2;
    m.bias = o; o += (64 + 128 + 4) * 4;          // bb0 | bb1 | b2
    m.total = o;
    return m;
}

// B operand (n = row0 + r, k) = w[r, k] for a weight w[rows_valid, k_valid] (row stride ld), panels of `rows` rows
__device__ __forceinline__ void stage_weight(uint8_t* hi, uint8_t* lo, const float* __restrict__ w, int64_t ld, int rows,
                                             int rows_valid, int k_valid, int row0, int tid) {
    for (int e = tid; e < rows_valid * k_valid; e += THREADS) {
        const int r = e / k_valid, k = e - r * k_valid;
        float h, l;
        split(__ldg(w + (int64_t)r * ld + k), h, l);
        const int off = b_off(row0 + r, k, rows);
        *reinterpret_cast<float*>(hi + off) = h;
        *reinterpret_cast<float*>(lo + off) = l;
    }
}
// B operand (n = row0 + j, k = o) = w[o, j]: the transposed weight of a data gradient
__device__ __forceinline__ void stage_weight_t(uint8_t* hi, uint8_t* lo, const float* __restrict__ w, int64_t ld, int rows,
                                               int rows_valid, int k_valid, int row0, int tid) {
    for (int e = tid; e < rows_valid * k_valid; e += THREADS) {
        const int o = e / rows_valid, j = e - o * rows_valid;        // consecutive threads: consecutive j (coalesced)
        float h, l;
        split(__ldg(w + (int64_t)o * ld + j), h, l);
        const int off = b_off(row0 + j, o, rows);
        *reinterpret_cast<float*>(hi + off) = h;
        *reinterpret_cast<float*>(lo + off) = l;
    }
}

__device__ __forceinline__ float2 ld2(const float* p, bool ok) {
    return ok ? __ldg(reinterpret_cast<const float2*>(p)) : make_float2(0.f, 0.f);
}
__device__ __forceinline__ void st2(float* p, float a, float b, bool ok) {
    if (ok) *reinterpret_cast<float2*>(p) = make_float2(a, b);
}
// one step of (F_c + 0.5 F_f + 0.5 F_b) / 2 in torch's order: acc + 0.5 v, halved after the last query (no contraction)
__device__ __forceinline__ float blend(float acc, float v, bool last) {
    const float r = __fadd_rn(acc, __fmul_rn(0.5f, v));
    return last ? __fmul_rn(r, 0.5f) : r;
}
// Query qi's features (a, b) at dst folded into the running blend that this thread stored there for queries < qi
// (plain loads: the thread reads back its own stores); returns the stored pair.
__device__ __forceinline__ float2 blend_into(float* dst, float a, float b, int qi, bool last, bool ok) {
    if (qi > 0 && ok) {
        const float2 o = *reinterpret_cast<const float2*>(dst);
        a = blend(o.x, a, last);
        b = blend(o.y, b, last);
    }
    st2(dst, a, b, ok);
    return make_float2(a, b);
}

// dZ = acc * (saved > 0) on this thread's rows (saved and dst have row stride ld), stored, and split into the next A
__device__ __forceinline__ void relu_back(float (&acc)[32], const float* saved, float* dst, int64_t ld, int64_t row0,
                                          int64_t row1, bool ok0, bool ok1, int q, uint32_t (&ahi)[8][4],
                                          uint32_t (&alo)[8][4]) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const int c = 8 * j + 2 * q;
        const float2 m0 = ld2(saved + row0 * ld + c, ok0), m1 = ld2(saved + row1 * ld + c, ok1);
        acc[4 * j] = m0.x > 0.f ? acc[4 * j] : 0.f;
        acc[4 * j + 1] = m0.y > 0.f ? acc[4 * j + 1] : 0.f;
        acc[4 * j + 2] = m1.x > 0.f ? acc[4 * j + 2] : 0.f;
        acc[4 * j + 3] = m1.y > 0.f ? acc[4 * j + 3] : 0.f;
        st2(dst + row0 * ld + c, acc[4 * j], acc[4 * j + 1], ok0);
        st2(dst + row1 * ld + c, acc[4 * j + 2], acc[4 * j + 3], ok1);
        frag_split(acc[4 * j], acc[4 * j + 1], acc[4 * j + 2], acc[4 * j + 3], ahi[j], alo[j]);
    }
}

// Adds the column sums over the warp's 16 rows of a 64-column accumulator block to dst[0, 64).
__device__ __forceinline__ void ray_colsum(const float (&v)[32], float* dst, int lane, bool live) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            float s = v[4 * j + e] + v[4 * j + 2 + e];
            s += __shfl_xor_sync(0xffffffffu, s, 4);
            s += __shfl_xor_sync(0xffffffffu, s, 8);
            s += __shfl_xor_sync(0xffffffffu, s, 16);
            if (lane < 4 && live) atomicAdd(dst + 8 * j + 2 * lane + e, s);
        }
    }
}

// Q = 3: the flow variants' temporal aggregation (emer_flow_field_fwd).  Row i's three encodings are rows i, n + i and
// 2n + i of enc (current, forward-warped, backward-warped); each goes through the base MLP on its own, and the features
// blend as  feats = (F_c + 0.5 F_f + 0.5 F_b) / 2  (radiance_field.py:460, the same operation order) before the density
// and the colour head read them.  The running blend lives in the output rows (save_hg's geometry half, save_sem), each
// element read back by the thread that stored it while the tile is still in L2 (held in registers across the queries,
// it spills at <k, 64>); the last query's blend goes on in `feat`.  save_hb then holds 3n rows.  rgb == NULL (Q = 3
// only): density only, the colour head is skipped.
template <int K_ENC, int NF, int Q>
__device__ __forceinline__ void field_fwd_body(const FwdParams& p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const Smem m = smem_map(K_ENC, NF);
    float* bias_s = reinterpret_cast<float*>(smem + m.bias);
    const int tid = threadIdx.x;

    // ---- resident weights: zero the padded rows first (W2: rows 3..7), then split and scatter
    for (int i = tid * 16; i < m.bias; i += THREADS * 16) *reinterpret_cast<float4*>(smem + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    stage_weight(smem + m.wb0_hi, smem + m.wb0_lo, p.wb0, K_ENC, H, H, K_ENC, 0, tid);
    stage_weight(smem + m.wb1_hi, smem + m.wb1_lo, p.wb1, H, NF, NF, H, 0, tid);
    stage_weight(smem + m.wg_hi, smem + m.wg_lo, p.w0g, p.ld_w0, 128, H, H, 0, tid);
    stage_weight(smem + m.wg_hi, smem + m.wg_lo, p.w1g, p.ld_w1, 128, H, H, H, tid);
    stage_weight(smem + m.w1h_hi, smem + m.w1h_lo, p.w1h, p.ld_w1, H, H, H, 0, tid);
    stage_weight(smem + m.w2_hi, smem + m.w2_lo, p.w2, H, 8, 3, H, 0, tid);
    for (int e = tid; e < 64 + 128 + 4; e += THREADS) {
        float v = 0.0f;
        if (e < 64) v = __ldg(p.bb0 + e);
        else if (e < 64 + 128) { if (e - 64 < NF) v = __ldg(p.bb1 + e - 64); }
        else if (e - 192 < 3) v = __ldg(p.b2 + e - 192);
        bias_s[e] = v;
    }
    fence_async_proxy();
    __syncthreads();

    const uint32_t sb = smem_u32(smem);
    const int wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
    const float* bb0_s = bias_s;
    const float* bb1_s = bias_s + 64;
    const float* b2_s = bias_s + 192;
    const int64_t n_tiles = (p.n + ROWS - 1) / ROWS;

    for (int64_t tile = (int64_t)blockIdx.x * WGS + wg; tile < n_tiles; tile += (int64_t)gridDim.x * WGS) {
        const int64_t row0 = tile * ROWS + 16 * w + (lane >> 2), row1 = row0 + 8;
        const bool ok0 = row0 < p.n, ok1 = row1 < p.n;
        uint32_t ahi[8][4], alo[8][4];
        float feat[32];                       // the (blended) geometry features, this thread's rows and columns
#pragma unroll 1
        for (int qi = 0; qi < Q; ++qi) {
            const int64_t qo = (int64_t)qi * p.n;   // query qi's first row

            // ---- stage 0: Hb = relu(enc Wb0^T + bb0)
            // Rows past n read row n - 1 instead: a per-lane conditional load feeding the A operand makes ptxas serialize
            // every wgmma of the kernel (C7520).  Rows of a tile are independent and rows >= n are never stored.
            const float* x0p = p.enc + (qo + (ok0 ? row0 : p.n - 1)) * p.ld_enc + 2 * q;
            const float* x1p = p.enc + (qo + (ok1 ? row1 : p.n - 1)) * p.ld_enc + 2 * q;
#pragma unroll
            for (int j = 0; j < K_ENC / 8; ++j) {
                const float2 x0 = __ldg(reinterpret_cast<const float2*>(x0p + 8 * j));
                const float2 x1 = __ldg(reinterpret_cast<const float2*>(x1p + 8 * j));
                frag_split(x0.x, x0.y, x1.x, x1.y, ahi[j], alo[j]);
            }
            float acc[32];
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < K_ENC / 8; ++ks)
                mma3<64>(acc, ahi[ks], alo[ks], b_desc(sb + m.wb0_hi, H, ks, 0), b_desc(sb + m.wb0_lo, H, ks, 0), ks > 0);
            wg_commit();
            wg_wait0();
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = 8 * j + 2 * q;
                const float v0 = fmaxf(acc[4 * j] + bb0_s[c], 0.0f), v1 = fmaxf(acc[4 * j + 1] + bb0_s[c + 1], 0.0f);
                const float v2 = fmaxf(acc[4 * j + 2] + bb0_s[c], 0.0f), v3 = fmaxf(acc[4 * j + 3] + bb0_s[c + 1], 0.0f);
                if (p.save_hb) {
                    st2(p.save_hb + (qo + row0) * H + c, v0, v1, ok0);
                    st2(p.save_hb + (qo + row1) * H + c, v2, v3, ok1);
                }
                frag_split(v0, v1, v2, v3, ahi[j], alo[j]);
            }

            // ---- stage 1: feats = Hb Wb1^T + bb1; sigma = exp(feats[0] - 1); geo -> operand; semantic half -> HBM
            // The semantic half goes first, on its own: with both halves in flight at once <k,128> spills.
            if constexpr (NF > H) {
                float sem[32];
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks)
                    mma3<64>(sem, ahi[ks], alo[ks], b_desc(sb + m.wb1_hi, NF, ks, H), b_desc(sb + m.wb1_lo, NF, ks, H), ks > 0);
                wg_commit();
                wg_wait0();
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + 2 * q;
                    const float s0 = sem[4 * j] + bb1_s[H + c], s1 = sem[4 * j + 1] + bb1_s[H + c + 1];
                    const float s2 = sem[4 * j + 2] + bb1_s[H + c], s3 = sem[4 * j + 3] + bb1_s[H + c + 1];
                    blend_into(p.save_sem + row0 * H + c, s0, s1, qi, qi == Q - 1, ok0);
                    blend_into(p.save_sem + row1 * H + c, s2, s3, qi, qi == Q - 1, ok1);
                }
            }
            float geo[32];
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks)
                mma3<64>(geo, ahi[ks], alo[ks], b_desc(sb + m.wb1_hi, NF, ks, 0), b_desc(sb + m.wb1_lo, NF, ks, 0), ks > 0);
            wg_commit();
            wg_wait0();
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int c = 8 * j + 2 * q;
                const float v0 = geo[4 * j] + bb1_s[c], v1 = geo[4 * j + 1] + bb1_s[c + 1];
                const float v2 = geo[4 * j + 2] + bb1_s[c], v3 = geo[4 * j + 3] + bb1_s[c + 1];
                if constexpr (Q > 1) {
                    const float2 f0 = blend_into(p.save_hg + row0 * 128 + H + c, v0, v1, qi, qi == Q - 1, ok0);
                    const float2 f1 = blend_into(p.save_hg + row1 * 128 + H + c, v2, v3, qi, qi == Q - 1, ok1);
                    feat[4 * j] = f0.x; feat[4 * j + 1] = f0.y; feat[4 * j + 2] = f1.x; feat[4 * j + 3] = f1.y;
                } else {
                    feat[4 * j] = v0; feat[4 * j + 1] = v1; feat[4 * j + 2] = v2; feat[4 * j + 3] = v3;
                }
            }
        }  // queries
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + 2 * q;
            const float v0 = feat[4 * j], v1 = feat[4 * j + 1], v2 = feat[4 * j + 2], v3 = feat[4 * j + 3];
            if (j == 0 && q == 0) {
                if (ok0) p.sigma[row0] = density_fwd(v0);
                if (ok1) p.sigma[row1] = density_fwd(v2);
            }
            if (Q == 1 && p.save_hg) {
                st2(p.save_hg + row0 * 128 + H + c, v0, v1, ok0);
                st2(p.save_hg + row1 * 128 + H + c, v2, v3, ok1);
            }
            frag_split(v0, v1, v2, v3, ahi[j], alo[j]);
        }

        if constexpr (Q > 1) {
            if (!p.rgb) continue;             // density only
        }

        // ---- stage 2: [pre-h0 | partial h1] = G [W0g; W1g]^T;  H0 = relu(pre-h0 + ray_bias0)
        float d0[32], d1[32];
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks) {
            mma3<64>(d0, ahi[ks], alo[ks], b_desc(sb + m.wg_hi, 128, ks, 0), b_desc(sb + m.wg_lo, 128, ks, 0), ks > 0);
            mma3<64>(d1, ahi[ks], alo[ks], b_desc(sb + m.wg_hi, 128, ks, H), b_desc(sb + m.wg_lo, 128, ks, H), ks > 0);
        }
        wg_commit();
        wg_wait0();
        const float* rb0 = p.ray_bias + ((ok0 ? row0 : p.n - 1) / p.samples) * 128;
        const float* rb1 = p.ray_bias + ((ok1 ? row1 : p.n - 1) / p.samples) * 128;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + 2 * q;
            const float2 b0 = __ldg(reinterpret_cast<const float2*>(rb0 + c)), b1 = __ldg(reinterpret_cast<const float2*>(rb1 + c));
            const float v0 = fmaxf(d0[4 * j] + b0.x, 0.0f), v1 = fmaxf(d0[4 * j + 1] + b0.y, 0.0f);
            const float v2 = fmaxf(d0[4 * j + 2] + b1.x, 0.0f), v3 = fmaxf(d0[4 * j + 3] + b1.y, 0.0f);
            if (p.save_hg) {
                st2(p.save_hg + row0 * 128 + c, v0, v1, ok0);
                st2(p.save_hg + row1 * 128 + c, v2, v3, ok1);
            }
            frag_split(v0, v1, v2, v3, ahi[j], alo[j]);
        }

        // ---- stage 3: H1 = relu(partial h1 + H0 W1h^T + ray_bias1)
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)
            mma3<64>(d1, ahi[ks], alo[ks], b_desc(sb + m.w1h_hi, H, ks, 0), b_desc(sb + m.w1h_lo, H, ks, 0), 1);
        wg_commit();
        wg_wait0();
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + 2 * q;
            const float2 b0 = __ldg(reinterpret_cast<const float2*>(rb0 + H + c));
            const float2 b1 = __ldg(reinterpret_cast<const float2*>(rb1 + H + c));
            const float v0 = fmaxf(d1[4 * j] + b0.x, 0.0f), v1 = fmaxf(d1[4 * j + 1] + b0.y, 0.0f);
            const float v2 = fmaxf(d1[4 * j + 2] + b1.x, 0.0f), v3 = fmaxf(d1[4 * j + 3] + b1.y, 0.0f);
            if (p.save_h1) {
                st2(p.save_h1 + row0 * H + c, v0, v1, ok0);
                st2(p.save_h1 + row1 * H + c, v2, v3, ok1);
            }
            frag_split(v0, v1, v2, v3, ahi[j], alo[j]);
        }

        // ---- stage 4: rgb = sigmoid(H1 W2^T + b2)   (columns 2q, 2q + 1: quads 0 and 1 hold the three outputs)
        float d2[4];
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < 8; ++ks)
            mma3<8>(d2, ahi[ks], alo[ks], b_desc(sb + m.w2_hi, 8, ks, 0), b_desc(sb + m.w2_lo, 8, ks, 0), ks > 0);
        wg_commit();
        wg_wait0();
#pragma unroll
        for (int e = 0; e < 2; ++e) {
            const int c = 2 * q + e;
            if (c < 3) {
                if (ok0) p.rgb[row0 * 3 + c] = 1.0f / (1.0f + expf(-(d2[e] + b2_s[c])));
                if (ok1) p.rgb[row1 * 3 + c] = 1.0f / (1.0f + expf(-(d2[2 + e] + b2_s[c])));
            }
        }
    }
}


// ------------------------------------------------------------------------------------------------------------------
// Backward, data path: the gradient walks the same chain, again with every intermediate in registers.
//
//   dZ2 = d_rgb * rgb (1 - rgb)                                        (registers)
//   s0  dH1 = dZ2 W2                 A = dZ2 [.. x 8]   B = W2^T   [64 x 8]     dZ1 = dH1 * (h1 > 0)      -> HBM, operand
//   s1  [dH0 | dG] = dZ1 [W1h | W1g] A = dZ1            B = W1hg^T [128 x 64]   dZ0 = dH0 * (h0 > 0)      -> HBM, operand
//   s2  dG += dZ0 W0g                A = dZ0            B = W0g^T  [64 x 64]    dF = dG + d_geo, dF[0] += d_sigma * min(sigma, e^15)
//   s3  dHb = dF Wb1 (+ d_sem Wb1s)  A = dF (, d_sem)   B = Wb1^T  [64 x nf]    dZb = dHb * (hb > 0)      -> HBM, operand
//   s4  d_enc = dZb Wb0              A = dZb            B = Wb0^T  [k_enc x 64]                           -> HBM
//
// dZ1, [dZ0 | dF], dZb are written out because the weight gradients (X^T dZ over ALL rows, wgrad_mn.cu) read them; the
// per-ray sums of dZ0 / dZ1 -- the gradient of the per-ray bias, i.e. of the direction / embedding columns of the head --
// are reduced here with warp shuffles (a warp's 16 rows are consecutive samples of one ray) and added to d_ray_bias[R, 128].
struct BwdParams {
    const float *d_rgb, *rgb, *d_sigma, *sigma, *d_geo, *d_sem;      // [N,3] [N,3] [N] [N] [N,64]|null [N,64]|null
    const float *hb, *hg, *h1;                                       // saved activations [N,64] [N,128] [N,64]
    const float *wb0, *wb1; int n_feat;                              // [64, k_enc], [n_feat, 64]
    const float* w0g; int64_t ld_w0; const float *w1h, *w1g; int64_t ld_w1; const float* w2;
    float *dz2, *dz1, *d1, *dzb, *d_enc; int64_t ld_denc;            // [N,3], [N,64], [N,128] = [dZ0 | dF], [N,64], [N, k_enc]
    float* d_ray_bias; int samples;                                  // [R,128] += ; ray sums only when samples % 32 == 0
    float* d_sem_q;                                                  // Q = 3: [3N,64] the three queries' d_sem | null
    int64_t n;
};

struct BSmem {
    int w2_hi, w2_lo, w1_hi, w1_lo, w0_hi, w0_lo, wb1_hi, wb1_lo, wb0_hi, wb0_lo, total;
};
__host__ __device__ inline BSmem bsmem_map(int k_enc, int n_feat) {
    BSmem m;
    int o = 0;
    const int w2 = (8 / 4) * H * 16, w1 = (H / 4) * 128 * 16, w0 = (H / 4) * H * 16, wb1 = (n_feat / 4) * H * 16,
              wb0 = (H / 4) * k_enc * 16;
    m.w2_hi = o; o += w2; m.w2_lo = o; o += w2;
    m.w1_hi = o; o += w1; m.w1_lo = o; o += w1;
    m.w0_hi = o; o += w0; m.w0_lo = o; o += w0;
    m.wb1_hi = o; o += wb1; m.wb1_lo = o; o += wb1;
    m.wb0_hi = o; o += wb0; m.wb0_lo = o; o += wb0;
    m.total = o;
    return m;
}

// Q = 3 (emer_flow_field_bwd): the blended dF fans out to the three queries' base MLPs, scaled by the blend's
// d feats / d F_q = 1/2, 1/4, 1/4; dzb, d_enc and the dF half of d1 then hold 3n rows (current, forward, backward), and
// d_sem_q the scaled d_sem.  h1 == NULL (Q = 3 only): density only, the colour head's stages are skipped.
template <int K_ENC, int NF, int Q>
__device__ __forceinline__ void field_bwd_body(const BwdParams& p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const BSmem m = bsmem_map(K_ENC, NF);
    const int tid = threadIdx.x;
    for (int i = tid * 16; i < m.total; i += THREADS * 16) *reinterpret_cast<float4*>(smem + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    stage_weight_t(smem + m.w2_hi, smem + m.w2_lo, p.w2, H, H, H, 3, 0, tid);                  // [64 x 8]
    stage_weight_t(smem + m.w1_hi, smem + m.w1_lo, p.w1h, p.ld_w1, 128, H, H, 0, tid);         // rows 0..63
    stage_weight_t(smem + m.w1_hi, smem + m.w1_lo, p.w1g, p.ld_w1, 128, H, H, H, tid);         // rows 64..127
    stage_weight_t(smem + m.w0_hi, smem + m.w0_lo, p.w0g, p.ld_w0, H, H, H, 0, tid);
    stage_weight_t(smem + m.wb1_hi, smem + m.wb1_lo, p.wb1, H, H, H, NF, 0, tid);               // [64 x nf]
    stage_weight_t(smem + m.wb0_hi, smem + m.wb0_lo, p.wb0, K_ENC, K_ENC, K_ENC, H, 0, tid);    // [k_enc x 64]
    fence_async_proxy();
    __syncthreads();

    const uint32_t sb = smem_u32(smem);
    const int wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
    const bool ray_sums = p.d_ray_bias != nullptr && (p.samples % 32 == 0);
    const int64_t n_tiles = (p.n + ROWS - 1) / ROWS;

    for (int64_t tile = (int64_t)blockIdx.x * WGS + wg; tile < n_tiles; tile += (int64_t)gridDim.x * WGS) {
        const int64_t wrow0 = tile * ROWS + 16 * w;                     // the warp's first row
        const int64_t row0 = wrow0 + (lane >> 2), row1 = row0 + 8;
        const bool ok0 = row0 < p.n, ok1 = row1 < p.n;
        // the warp's 16 rows belong to one ray (samples % 32 == 0); rows past the end contribute zeros
        const bool warp_live = wrow0 < p.n;
        float* rbias = ray_sums ? p.d_ray_bias + (wrow0 / p.samples) * 128 : nullptr;
        uint32_t ahi[8][4], alo[8][4];
        float acc[32], dg[32];
        // (the flag read through a shuffle is visibly warp-uniform: otherwise ptxas serializes the wgmmas, C7520)
        const bool head = Q == 1 || __shfl_sync(0xffffffffu, (int)(p.h1 != nullptr), 0) != 0;
        if (head) {
            // ---- stage 0 operand: dZ2 = d_rgb * rgb (1 - rgb), columns 2q, 2q + 1 of one 8-wide k step
            {
                float v[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const int c = 2 * q + (e & 1);
                    const int64_t row = (e < 2) ? row0 : row1;
                    if (c < 3 && (e < 2 ? ok0 : ok1) && p.d_rgb) {
                        const float y = __ldg(p.rgb + row * 3 + c);
                        v[e] = __ldg(p.d_rgb + row * 3 + c) * (y * (1.0f - y));
                        if (p.dz2) p.dz2[row * 3 + c] = v[e];
                    }
                }
                frag_split(v[0], v[1], v[2], v[3], ahi[0], alo[0]);
            }
            wg_fence();
            mma3<64>(acc, ahi[0], alo[0], b_desc(sb + m.w2_hi, H, 0, 0), b_desc(sb + m.w2_lo, H, 0, 0), 0);
            wg_commit();
            wg_wait0();

            // ---- stage 0 result: dZ1 = dH1 * (h1 > 0)
            relu_back(acc, p.h1, p.dz1, H, row0, row1, ok0, ok1, q, ahi, alo);
            if (ray_sums) ray_colsum(acc, rbias + H, lane, warp_live);

            // ---- stage 1: [dH0 | dG] = dZ1 [W1h | W1g];  dZ0 = dH0 * (h0 > 0)   (dG stays in its accumulator)
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks) {
                mma3<64>(acc, ahi[ks], alo[ks], b_desc(sb + m.w1_hi, 128, ks, 0), b_desc(sb + m.w1_lo, 128, ks, 0), ks > 0);
                mma3<64>(dg, ahi[ks], alo[ks], b_desc(sb + m.w1_hi, 128, ks, H), b_desc(sb + m.w1_lo, 128, ks, H), ks > 0);
            }
            wg_commit();
            wg_wait0();
            relu_back(acc, p.hg, p.d1, 128, row0, row1, ok0, ok1, q, ahi, alo);
            if (ray_sums) ray_colsum(acc, rbias, lane, warp_live);

            // ---- stage 2: dG += dZ0 W0g;  dF = dG (+ d_geo); dF[0] += d_sigma * exp(min(x, 15)), exp(x) = sigma (nerf_utils.py:72-75)
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks)
                mma3<64>(dg, ahi[ks], alo[ks], b_desc(sb + m.w0_hi, H, ks, 0), b_desc(sb + m.w0_lo, H, ks, 0), 1);
            wg_commit();
            wg_wait0();
        } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) dg[i] = 0.0f;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int c = 8 * j + 2 * q;
            float v0 = dg[4 * j], v1 = dg[4 * j + 1], v2 = dg[4 * j + 2], v3 = dg[4 * j + 3];
            if (p.d_geo) {
                const float2 g0 = ld2(p.d_geo + row0 * H + c, ok0), g1 = ld2(p.d_geo + row1 * H + c, ok1);
                v0 += g0.x; v1 += g0.y; v2 += g1.x; v3 += g1.y;
            }
            if (j == 0 && q == 0 && p.d_sigma) {
                if (ok0) v0 += __ldg(p.d_sigma + row0) * fminf(__ldg(p.sigma + row0), 3269017.25f);
                if (ok1) v2 += __ldg(p.d_sigma + row1) * fminf(__ldg(p.sigma + row1), 3269017.25f);
            }
            if constexpr (Q > 1) {
                dg[4 * j] = v0; dg[4 * j + 1] = v1; dg[4 * j + 2] = v2; dg[4 * j + 3] = v3;
            } else {
                st2(p.d1 + row0 * 128 + H + c, v0, v1, ok0);
                st2(p.d1 + row1 * 128 + H + c, v2, v3, ok1);
                frag_split(v0, v1, v2, v3, ahi[j], alo[j]);
            }
        }

#pragma unroll 1
        for (int qi = 0; qi < Q; ++qi) {
            const int64_t qo = (int64_t)qi * p.n;   // query qi's first row
            const float sq = qi == 0 ? 0.5f : 0.25f;  // d feats / d F_q (Q = 3)
            if constexpr (Q > 1) {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + 2 * q;
                    const float v0 = dg[4 * j] * sq, v1 = dg[4 * j + 1] * sq, v2 = dg[4 * j + 2] * sq, v3 = dg[4 * j + 3] * sq;
                    st2(p.d1 + (qo + row0) * 128 + H + c, v0, v1, ok0);
                    st2(p.d1 + (qo + row1) * 128 + H + c, v2, v3, ok1);
                    frag_split(v0, v1, v2, v3, ahi[j], alo[j]);
                }
            }

            // ---- stage 3: dHb = dF Wb1[:64] (+ d_sem Wb1[64:]);  dZb = dHb * (hb > 0)
            wg_fence();
#pragma unroll
            for (int ks = 0; ks < 8; ++ks)
                mma3<64>(acc, ahi[ks], alo[ks], b_desc(sb + m.wb1_hi, H, ks, 0), b_desc(sb + m.wb1_lo, H, ks, 0), ks > 0);
            wg_commit();
            wg_wait0();
            if constexpr (NF > H) {
                if (p.d_sem) {                           // the second operand piece: the gradient of the semantic half
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        const int c = 8 * j + 2 * q;
                        float2 s0 = ld2(p.d_sem + row0 * H + c, ok0), s1 = ld2(p.d_sem + row1 * H + c, ok1);
                        if constexpr (Q > 1) {
                            s0.x *= sq; s0.y *= sq; s1.x *= sq; s1.y *= sq;
                            st2(p.d_sem_q + (qo + row0) * H + c, s0.x, s0.y, ok0);
                            st2(p.d_sem_q + (qo + row1) * H + c, s1.x, s1.y, ok1);
                        }
                        frag_split(s0.x, s0.y, s1.x, s1.y, ahi[j], alo[j]);
                    }
                    wg_fence();
#pragma unroll
                    for (int ks = 0; ks < 8; ++ks)
                        mma3<64>(acc, ahi[ks], alo[ks], b_desc(sb + m.wb1_hi, H, 8 + ks, 0), b_desc(sb + m.wb1_lo, H, 8 + ks, 0), 1);
                    wg_commit();
                    wg_wait0();
                }
            }
            relu_back(acc, p.hb + qo * H, p.dzb + qo * H, H, row0, row1, ok0, ok1, q, ahi, alo);

            // ---- stage 4: d_enc = dZb Wb0
            if (p.d_enc) {
                float de[K_ENC / 2];
                wg_fence();
#pragma unroll
                for (int ks = 0; ks < 8; ++ks)
                    mma3<K_ENC>(de, ahi[ks], alo[ks], b_desc(sb + m.wb0_hi, K_ENC, ks, 0), b_desc(sb + m.wb0_lo, K_ENC, ks, 0), ks > 0);
                wg_commit();
                wg_wait0();
#pragma unroll
                for (int j = 0; j < K_ENC / 8; ++j) {
                    const int c = 8 * j + 2 * q;
                    st2(p.d_enc + (qo + row0) * p.ld_denc + c, de[4 * j], de[4 * j + 1], ok0);
                    st2(p.d_enc + (qo + row1) * p.ld_denc + c, de[4 * j + 2], de[4 * j + 3], ok1);
                }
            }
        }  // queries
    }
}

// The kernels: field_*_kernel<k_enc, n_feat> (one query per row) and, for the flow variants, flow_field_*_k<k>_f<nf>
// (three queries per row; no k_enc = 32: its backward's d_enc disagreed with fp64, and the flow configs' dynamic grid has
// L*F = 40).
template <int K_ENC, int NF>
__global__ void __launch_bounds__(THREADS, 1) field_fwd_kernel(const FwdParams p) { field_fwd_body<K_ENC, NF, 1>(p); }
template <int K_ENC, int NF>
__global__ void __launch_bounds__(THREADS, 1) field_bwd_kernel(const BwdParams p) { field_bwd_body<K_ENC, NF, 1>(p); }
#define EMER_FLOW_FIELD_KERNELS(K, NF)                                                                                   \
    __global__ void __launch_bounds__(THREADS, 1) flow_field_fwd_k##K##_f##NF(const FwdParams p) {                       \
        field_fwd_body<K, NF, 3>(p);                                                                                     \
    }                                                                                                                    \
    __global__ void __launch_bounds__(THREADS, 1) flow_field_bwd_k##K##_f##NF(const BwdParams p) {                       \
        field_bwd_body<K, NF, 3>(p);                                                                                     \
    }
EMER_FLOW_FIELD_KERNELS(40, 64)
EMER_FLOW_FIELD_KERNELS(40, 128)
EMER_FLOW_FIELD_KERNELS(64, 64)
EMER_FLOW_FIELD_KERNELS(64, 128)
#undef EMER_FLOW_FIELD_KERNELS

// kernel of (k_enc, n_feat, queries); k_enc = 32 has one query only
template <int K, int NF, int Q>
constexpr auto fwd_kernel() {
    if constexpr (Q == 1) return field_fwd_kernel<K, NF>;
    else if constexpr (K == 40 && NF == 64) return flow_field_fwd_k40_f64;
    else if constexpr (K == 40) return flow_field_fwd_k40_f128;
    else if constexpr (NF == 64) return flow_field_fwd_k64_f64;
    else return flow_field_fwd_k64_f128;
}
template <int K, int NF, int Q>
constexpr auto bwd_kernel() {
    if constexpr (Q == 1) return field_bwd_kernel<K, NF>;
    else if constexpr (K == 40 && NF == 64) return flow_field_bwd_k40_f64;
    else if constexpr (K == 40) return flow_field_bwd_k40_f128;
    else if constexpr (NF == 64) return flow_field_bwd_k64_f64;
    else return flow_field_bwd_k64_f128;
}

// One launcher per direction and query count: grid = min(SMs, tiles / WGS); the shared-memory attribute is set once per
// kernel and device.
template <int Q>
static int launch_fwd(const FwdParams& p, void* stream, const char* what) {
    const Smem m = smem_map(p.k_enc, p.n_feat);
    size_t smem = (size_t)m.total;
    EMER_REQUIRE(smem <= 227 * 1024, "%s: %zu B of shared memory needed", what, smem);
    const int64_t n_tiles = ceil_div(p.n, ROWS);
    int64_t grid = sm_count();
    if (grid > ceil_div(n_tiles, WGS)) grid = ceil_div(n_tiles, WGS);
    auto launch = [&](auto kernel, size_t& configured) -> int {
        if (smem > configured) {
            cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) {
                set_error("%s: cudaFuncSetAttribute(%zu): %s", what, smem, cudaGetErrorString(e));
                return -2;
            }
            configured = smem;
        }
        kernel<<<(unsigned)grid, THREADS, smem, (cudaStream_t)stream>>>(p);
        return 0;
    };
    static size_t configured_dev[6][64] = {{0}};          // the attribute is per kernel and per device
    const int dev = current_device();
    int rc;
    if (Q > 1 && p.k_enc == 32) {          // (no three-query instantiation at k_enc 32; the entry points refuse it)
        set_error("%s: k_enc=32", what);
        return -2;
    }
    if (p.n_feat == 64) {
        if (p.k_enc == 32) rc = launch(fwd_kernel<32, 64, 1>(), configured_dev[0][dev]);
        else if (p.k_enc == 40) rc = launch(fwd_kernel<40, 64, Q>(), configured_dev[1][dev]);
        else rc = launch(fwd_kernel<64, 64, Q>(), configured_dev[2][dev]);
    } else {
        if (p.k_enc == 32) rc = launch(fwd_kernel<32, 128, 1>(), configured_dev[3][dev]);
        else if (p.k_enc == 40) rc = launch(fwd_kernel<40, 128, Q>(), configured_dev[4][dev]);
        else rc = launch(fwd_kernel<64, 128, Q>(), configured_dev[5][dev]);
    }
    if (rc) return rc;
    return check_launch(what);
}

template <int Q>
static int launch_bwd(const BwdParams& p, int k_enc, void* stream, const char* what) {
    const BSmem m = bsmem_map(k_enc, p.n_feat);
    size_t smem = (size_t)m.total;
    EMER_REQUIRE(smem <= 227 * 1024, "%s: %zu B of shared memory needed", what, smem);
    const int64_t n_tiles = ceil_div(p.n, ROWS);
    int64_t grid = sm_count();
    if (grid > ceil_div(n_tiles, WGS)) grid = ceil_div(n_tiles, WGS);
    auto launch = [&](auto kernel, size_t& configured) -> int {
        if (smem > configured) {
            cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
            if (e != cudaSuccess) {
                set_error("%s: cudaFuncSetAttribute(%zu): %s", what, smem, cudaGetErrorString(e));
                return -2;
            }
            configured = smem;
        }
        kernel<<<(unsigned)grid, THREADS, smem, (cudaStream_t)stream>>>(p);
        return 0;
    };
    static size_t configured_dev[6][64] = {{0}};          // the attribute is per kernel and per device
    const int dev = current_device();
    int rc;
    if (Q > 1 && k_enc == 32) {          // (no three-query instantiation at k_enc 32; the entry points refuse it)
        set_error("%s: k_enc=32", what);
        return -2;
    }
    if (p.n_feat == 64) {
        if (k_enc == 32) rc = launch(bwd_kernel<32, 64, 1>(), configured_dev[0][dev]);
        else if (k_enc == 40) rc = launch(bwd_kernel<40, 64, Q>(), configured_dev[1][dev]);
        else rc = launch(bwd_kernel<64, 64, Q>(), configured_dev[2][dev]);
    } else {
        if (k_enc == 32) rc = launch(bwd_kernel<32, 128, 1>(), configured_dev[3][dev]);
        else if (k_enc == 40) rc = launch(bwd_kernel<40, 128, Q>(), configured_dev[4][dev]);
        else rc = launch(bwd_kernel<64, 128, Q>(), configured_dev[5][dev]);
    }
    if (rc) return rc;
    return check_launch(what);
}

}  // namespace ff
}  // namespace emer

using namespace emer;

extern "C" int emer_field_fwd(const float* enc, int64_t ld_enc, int k_enc, const float* wb0, const float* bb0,
                              const float* wb1, const float* bb1, int n_feat, const float* w0g, int64_t ld_w0,
                              const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, const float* b2,
                              const float* ray_bias, int samples, float* sigma, float* rgb, float* save_hb, float* save_hg,
                              float* save_h1, float* save_sem, int64_t n, void* stream) {
    using namespace emer::ff;
    if (n == 0) return 0;
    EMER_REQUIRE(enc && wb0 && bb0 && wb1 && bb1 && w0g && w1h && w1g && w2 && b2 && ray_bias && sigma && rgb,
                 "emer_field_fwd: NULL pointer");
    EMER_REQUIRE(k_enc == 32 || k_enc == 40 || k_enc == 64, "emer_field_fwd: k_enc=%d (L*F of the grid) must be 32, 40 or 64", k_enc);
    EMER_REQUIRE(n_feat == 64 || n_feat == 128, "emer_field_fwd: n_feat=%d must be 64 or 128", n_feat);
    EMER_REQUIRE(samples > 0, "emer_field_fwd: samples per ray must be positive");
    EMER_REQUIRE(ld_enc % 8 == 0 && ((uintptr_t)enc & 31) == 0, "emer_field_fwd: enc rows must be 32-byte aligned");
    EMER_REQUIRE(((uintptr_t)ray_bias & 15) == 0, "emer_field_fwd: ray_bias must be 16-byte aligned");
    EMER_REQUIRE((((uintptr_t)save_hb | (uintptr_t)save_hg | (uintptr_t)save_h1 | (uintptr_t)save_sem) & 31) == 0,
                 "emer_field_fwd: save buffers must be 32-byte aligned");
    EMER_REQUIRE(n_feat == 64 || save_sem, "emer_field_fwd: the semantic half needs its output buffer");
    FwdParams p{};
    p.enc = enc; p.ld_enc = ld_enc; p.k_enc = k_enc; p.wb0 = wb0; p.bb0 = bb0; p.wb1 = wb1; p.bb1 = bb1; p.n_feat = n_feat;
    p.w0g = w0g; p.ld_w0 = ld_w0; p.w1h = w1h; p.w1g = w1g; p.ld_w1 = ld_w1; p.w2 = w2; p.b2 = b2;
    p.ray_bias = ray_bias; p.samples = samples; p.sigma = sigma; p.rgb = rgb;
    p.save_hb = save_hb; p.save_hg = save_hg; p.save_h1 = save_h1; p.save_sem = save_sem; p.n = n;
    return launch_fwd<1>(p, stream, "emer_field_fwd");
}

extern "C" int emer_field_bwd(const float* d_rgb, const float* rgb, const float* d_sigma, const float* sigma,
                              const float* d_geo, const float* d_sem, const float* hb, const float* hg, const float* h1,
                              const float* wb0, int k_enc, const float* wb1, int n_feat, const float* w0g, int64_t ld_w0,
                              const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, float* dz2, float* dz1,
                              float* d1, float* dzb, float* d_enc, int64_t ld_denc, float* d_ray_bias, int samples,
                              int64_t n, void* stream) {
    using namespace emer::ff;
    if (n == 0) return 0;
    EMER_REQUIRE(rgb && sigma && hb && hg && h1 && wb0 && wb1 && w0g && w1h && w1g && w2 && dz1 && d1 && dzb,
                 "emer_field_bwd: NULL pointer");
    EMER_REQUIRE(k_enc == 32 || k_enc == 40 || k_enc == 64, "emer_field_bwd: k_enc=%d must be 32, 40 or 64", k_enc);
    EMER_REQUIRE(n_feat == 64 || n_feat == 128, "emer_field_bwd: n_feat=%d must be 64 or 128", n_feat);
    EMER_REQUIRE(samples > 0, "emer_field_bwd: samples per ray must be positive");
    EMER_REQUIRE(!d_enc || (ld_denc % 8 == 0 && ld_denc >= k_enc), "emer_field_bwd: d_enc rows must be 32-byte aligned");
    EMER_REQUIRE((((uintptr_t)hb | (uintptr_t)hg | (uintptr_t)h1 | (uintptr_t)dz1 | (uintptr_t)d1 | (uintptr_t)dzb |
                   (uintptr_t)d_enc | (uintptr_t)d_geo | (uintptr_t)d_sem) & 31) == 0,
                 "emer_field_bwd: row buffers must be 32-byte aligned");
    EMER_REQUIRE(!d_ray_bias || samples % 32 == 0, "emer_field_bwd: per-ray sums need samples %% 32 == 0 (got %d)", samples);
    BwdParams p{};
    p.d_rgb = d_rgb; p.rgb = rgb; p.d_sigma = d_sigma; p.sigma = sigma; p.d_geo = d_geo; p.d_sem = d_sem;
    p.hb = hb; p.hg = hg; p.h1 = h1; p.wb0 = wb0; p.wb1 = wb1; p.n_feat = n_feat;
    p.w0g = w0g; p.ld_w0 = ld_w0; p.w1h = w1h; p.w1g = w1g; p.ld_w1 = ld_w1; p.w2 = w2;
    p.dz2 = dz2; p.dz1 = dz1; p.d1 = d1; p.dzb = dzb; p.d_enc = d_enc; p.ld_denc = ld_denc; p.d_ray_bias = d_ray_bias; p.samples = samples;
    p.n = n;
    return launch_bwd<1>(p, k_enc, stream, "emer_field_bwd");
}

extern "C" int emer_flow_field_fwd(const float* enc, int64_t ld_enc, int k_enc, const float* wb0, const float* bb0,
                                   const float* wb1, const float* bb1, int n_feat, const float* w0g, int64_t ld_w0,
                                   const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, const float* b2,
                                   const float* ray_bias, int samples, float* sigma, float* rgb, float* save_hb,
                                   float* save_hg, float* save_h1, float* save_sem, int64_t n, void* stream) {
    using namespace emer::ff;
    if (n == 0) return 0;
    EMER_REQUIRE(enc && wb0 && bb0 && wb1 && bb1 && w0g && w1h && w1g && w2 && b2 && sigma,
                 "emer_flow_field_fwd: NULL pointer");
    EMER_REQUIRE(!rgb || ray_bias, "emer_flow_field_fwd: the colour head needs ray_bias");
    EMER_REQUIRE(k_enc == 40 || k_enc == 64, "emer_flow_field_fwd: k_enc=%d must be 40 or 64", k_enc);
    EMER_REQUIRE(n_feat == 64 || n_feat == 128, "emer_flow_field_fwd: n_feat=%d must be 64 or 128", n_feat);
    EMER_REQUIRE(samples > 0, "emer_flow_field_fwd: samples per ray must be positive");
    EMER_REQUIRE(ld_enc % 8 == 0 && ((uintptr_t)enc & 31) == 0, "emer_flow_field_fwd: enc rows must be 32-byte aligned");
    EMER_REQUIRE(((uintptr_t)ray_bias & 15) == 0, "emer_flow_field_fwd: ray_bias must be 16-byte aligned");
    EMER_REQUIRE((((uintptr_t)save_hb | (uintptr_t)save_hg | (uintptr_t)save_h1 | (uintptr_t)save_sem) & 31) == 0,
                 "emer_flow_field_fwd: save buffers must be 32-byte aligned");
    EMER_REQUIRE(save_hg && (n_feat == 64 || save_sem), "emer_flow_field_fwd: the blend needs save_hg (and save_sem at n_feat 128)");
    EMER_REQUIRE(n <= INT64_MAX / 3 / ld_enc, "emer_flow_field_fwd: n=%lld too large", (long long)n);
    FwdParams p{};
    p.enc = enc; p.ld_enc = ld_enc; p.k_enc = k_enc; p.wb0 = wb0; p.bb0 = bb0; p.wb1 = wb1; p.bb1 = bb1; p.n_feat = n_feat;
    p.w0g = w0g; p.ld_w0 = ld_w0; p.w1h = w1h; p.w1g = w1g; p.ld_w1 = ld_w1; p.w2 = w2; p.b2 = b2;
    p.ray_bias = ray_bias; p.samples = samples; p.sigma = sigma; p.rgb = rgb;
    p.save_hb = save_hb; p.save_hg = save_hg; p.save_h1 = save_h1; p.save_sem = save_sem; p.n = n;
    return launch_fwd<3>(p, stream, "emer_flow_field_fwd");
}

extern "C" int emer_flow_field_bwd(const float* d_rgb, const float* rgb, const float* d_sigma, const float* sigma,
                                   const float* d_geo, const float* d_sem, const float* hb, const float* hg,
                                   const float* h1, const float* wb0, int k_enc, const float* wb1, int n_feat,
                                   const float* w0g, int64_t ld_w0, const float* w1h, const float* w1g, int64_t ld_w1,
                                   const float* w2, float* dz2, float* dz1, float* d1, float* dzb, float* d_enc,
                                   int64_t ld_denc, float* d_ray_bias, float* d_sem_q, int samples, int64_t n,
                                   void* stream) {
    using namespace emer::ff;
    if (n == 0) return 0;
    const bool head = h1 != nullptr;
    EMER_REQUIRE(sigma && hb && wb0 && wb1 && w0g && w1h && w1g && w2 && d1 && dzb, "emer_flow_field_bwd: NULL pointer");
    EMER_REQUIRE(!head || (rgb && hg && dz1), "emer_flow_field_bwd: NULL pointer among the colour head's buffers");
    EMER_REQUIRE(head || (!d_rgb && !d_ray_bias && !dz2), "emer_flow_field_bwd: density only (h1 == NULL) takes no colour gradient");
    EMER_REQUIRE(!d_sem || d_sem_q, "emer_flow_field_bwd: d_sem needs d_sem_q");
    EMER_REQUIRE(k_enc == 40 || k_enc == 64, "emer_flow_field_bwd: k_enc=%d must be 40 or 64", k_enc);
    EMER_REQUIRE(n_feat == 64 || n_feat == 128, "emer_flow_field_bwd: n_feat=%d must be 64 or 128", n_feat);
    EMER_REQUIRE(samples > 0, "emer_flow_field_bwd: samples per ray must be positive");
    EMER_REQUIRE(!d_enc || (ld_denc % 8 == 0 && ld_denc >= k_enc), "emer_flow_field_bwd: d_enc rows must be 32-byte aligned");
    EMER_REQUIRE((((uintptr_t)hb | (uintptr_t)hg | (uintptr_t)h1 | (uintptr_t)dz1 | (uintptr_t)d1 | (uintptr_t)dzb |
                   (uintptr_t)d_enc | (uintptr_t)d_geo | (uintptr_t)d_sem | (uintptr_t)d_sem_q) & 31) == 0,
                 "emer_flow_field_bwd: row buffers must be 32-byte aligned");
    EMER_REQUIRE(!d_ray_bias || samples % 32 == 0, "emer_flow_field_bwd: per-ray sums need samples %% 32 == 0 (got %d)", samples);
    BwdParams p{};
    p.d_rgb = d_rgb; p.rgb = rgb; p.d_sigma = d_sigma; p.sigma = sigma; p.d_geo = d_geo; p.d_sem = d_sem;
    p.hb = hb; p.hg = hg; p.h1 = h1; p.wb0 = wb0; p.wb1 = wb1; p.n_feat = n_feat;
    p.w0g = w0g; p.ld_w0 = ld_w0; p.w1h = w1h; p.w1g = w1g; p.ld_w1 = ld_w1; p.w2 = w2;
    p.dz2 = dz2; p.dz1 = dz1; p.d1 = d1; p.dzb = dzb; p.d_enc = d_enc; p.ld_denc = ld_denc; p.d_ray_bias = d_ray_bias; p.samples = samples;
    p.d_sem_q = d_sem_q; p.n = n;
    return launch_bwd<3>(p, k_enc, stream, "emer_flow_field_bwd");
}
