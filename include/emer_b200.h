/*
 * emer_b200 -- C ABI of the H100-native EmerNeRF hot path (libemer_b200.so, sm_90a only).
 *
 * This is the drop-in boundary.  The reference reaches its native code through two Python
 * FFIs: the tiny-cuda-nn pybind object (third_party/tcnn_modules.py:102,122,161,216-219) and
 * nerfacc's `_C` extension (third_party/nerfacc_prop_net.py:11-14,153,172;
 * radiance_fields/render_utils.py:4-8).  Every entry point below names the reference call it
 * replaces.  The fused entry points (emer_mlp_*, emer_composite_*) replace chains of torch
 * library calls on the same path (radiance_fields/mlp.py:38-46, radiance_field.py:74-198,
 * render_utils.py:73-115).
 *
 * Conventions
 *   - all pointers are DEVICE pointers into caller-owned (PyTorch caching-allocator) memory,
 *     fp32 unless noted, dense row-major; the library allocates nothing on the hot path
 *   - `stream` is a cudaStream_t passed as void*; calls are asynchronous, re-entrant per stream,
 *     and never synchronise the host
 *   - return 0 on success; on failure a negative code, with emer_last_error() giving the text.
 *     No exceptions cross the boundary.  Shape/dtype/contiguity are validated by the caller
 *     (emernerf_b200/_ops.py), mirroring third_party/tcnn_modules.py:236-262.
 */
#ifndef EMER_B200_H
#define EMER_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EMER_MAX_LEVELS 16

/* Level table of one multi-resolution grid (host struct, passed by pointer, copied per launch).
 * Replaces the opaque object returned by _C.create_encoding(n_input_dims, encoding_config,
 * precision) -- third_party/tcnn_modules.py:420-423.  Filled by emernerf_b200/grid_desc.py with
 * tiny-cuda-nn's level formulas (scale_l = exp2(l*log2(per_level_scale))*base - 1,
 * res_l = ceil(scale_l)+1, size_l = min(round_up(res^D, 8), 2^log2_hashmap_size)). */
typedef struct emer_grid_desc {
    int32_t n_dims;                          /* 3 or 4 */
    int32_t n_levels;                        /* 1..16 */
    int32_t n_feat;                          /* 1, 2 or 4 floats per entry */
    int32_t reserved;
    float scale[EMER_MAX_LEVELS];
    uint32_t resolution[EMER_MAX_LEVELS];
    uint32_t offset[EMER_MAX_LEVELS + 1];    /* in entries; level l owns [offset[l], offset[l+1]) */
    uint32_t hashed[EMER_MAX_LEVELS];        /* 1: coherent-prime hash, 0: dense stride index */
} emer_grid_desc;

const char* emer_last_error(void);
int emer_version(void);

/* ---- multi-resolution hash grid (replaces native_tcnn_module.fwd / .bwd,
 *      third_party/tcnn_modules.py:122,161) ------------------------------------------------- */
/* y[N, L*F] = encode(x[N, D]); feature index = level*F + f. */
int emer_grid_fwd(const emer_grid_desc* g, const float* x, const float* table, float* y,
                  int64_t n, void* stream);
/* dtable (same layout as table, ACCUMULATED with atomics -- caller zeroes) and/or dx[N, D];
 * either may be NULL. */
int emer_grid_bwd(const emer_grid_desc* g, const float* x, const float* table, const float* dy,
                  float* dtable, float* dx, int64_t n, void* stream);
/* test hook: corner entry indices [N, L, 2^D] (int32, absolute entry index) -- the "bit-exact
 * sample indices" check of BASELINE.json. */
int emer_grid_indices(const emer_grid_desc* g, const float* x, int32_t* idx, int64_t n, void* stream);

/* ---- scene contraction (radiance_fields/nerf_utils.py:13-28 + the 0/1 selector of
 *      radiance_field.py:294-300,834-835) ----------------------------------------------------- */
/* out[N, out_dim] (out_dim 3 or 4): columns 0..2 = contracted*selector; column 3 = time[N]
 * (broadcast per point) when out_dim == 4.  unbounded=0 -> plain aabb normalisation.
 * apply_selector=0 gives the bare `contract()` of nerf_utils.py (no zeroing of outside points). */
int emer_contract_fwd(const float* pos, const float* aabb6, const float* time, float* out,
                      int out_dim, int unbounded, int apply_selector, int64_t n, void* stream);
/* dpos[N,3] = J^T dout[:, 0:3] (selector and time carry no gradient to pos; dtime_or_null[N]
 * receives dout[:,3]). */
int emer_contract_bwd(const float* pos, const float* aabb6, const float* dout, float* dpos,
                      float* dtime, int out_dim, int unbounded, int apply_selector, int64_t n,
                      void* stream);

/* ---- density activation trunc_exp(x - 1) (radiance_fields/nerf_utils.py:59-75,
 *      radiance_field.py:28,794).  x has row stride ldx (reads column 0). ------------------- */
int emer_trunc_exp_fwd(const float* x, int64_t ldx, float* y, int64_t n, void* stream);
int emer_trunc_exp_bwd(const float* x, int64_t ldx, const float* dy, float* dx, int64_t n, void* stream);

/* ---- dense layers of the MLP heads (replaces cuBLAS SGEMM under nn.Linear:
 *      radiance_fields/mlp.py:38-46, radiance_field.py:74-198,808-812) ---------------------- */
enum { EMER_ACT_NONE = 0, EMER_ACT_RELU = 1, EMER_ACT_SIGMOID = 2 };
/* Y[N, n_out] = act(X[N, k] W[n_out, k]^T + b) */
int emer_linear_fwd(const float* x, int64_t ldx, const float* w, const float* b, float* y,
                    int64_t ldy, int64_t n, int k, int n_out, int act, void* stream);
/* dZ = dY * act'(Y);  dX[N, k] (=|+=) dZ W */
int emer_linear_bwd_data(const float* dy, int64_t lddy, const float* y, int64_t ldy, int act,
                         const float* w, float* dx, int64_t lddx, int64_t n, int k, int n_out,
                         int accumulate, void* stream);
/* dW[n_out, k] += dZ^T X;  db[n_out] += sum_rows dZ   (atomics; caller zeroes) */
int emer_linear_bwd_weight(const float* x, int64_t ldx, const float* dy, int64_t lddy,
                           const float* y, int64_t ldy, int act, float* dw, float* db,
                           int64_t n, int k, int n_out, void* stream);

/* Narrow heads (n_out <= 8, k <= 256: rgb 64->3, density 64->1, flow 64->6, shadow 64->1): streaming
 * FFMA kernels; bwd_data fuses the ReLU mask of the layer below like the tensor-core kernel. */
int emer_linear_narrow_fwd(const float* x, int64_t ldx, const float* w, const float* b, float* y,
                           int64_t ldy, int64_t n, int k, int n_out, int act, void* stream);
int emer_linear_narrow_bwd_data(const float* dz, int64_t lddz, const float* w, float* dx, int64_t lddx,
                                const float* relu_src, int64_t ld_relu, int relu_cols, int64_t n, int k,
                                int n_out, void* stream);
int emer_linear_narrow_bwd_weight(const float* x, int64_t ldx, const float* dz, int64_t lddz, float* dw,
                                  float* db, int64_t n, int k, int n_out, void* stream);

/* Same contracts on the tensor cores: fp32 operands split into tf32 hi+lo, three
 * wgmma.mma_async ...tf32 per k-step accumulate A_hi*B_hi + A_lo*B_hi + A_hi*B_lo in registers
 * (fp32-accurate "3xTF32"; see emernerf_b200/csrc/linear_tc.cu).  Widths: k, n_out <= 256. */
int emer_linear_tc_fwd(const float* x, int64_t ldx, const float* w, const float* b, float* y,
                       int64_t ldy, int64_t n, int k, int n_out, int act, void* stream);
int emer_linear_tc_bwd_data(const float* dy, int64_t lddy, const float* y, int64_t ldy, int act,
                            const float* w, float* dx, int64_t lddx, const float* relu_src,
                            int64_t ld_relu, int relu_cols, int64_t n, int k, int n_out,
                            int accumulate, void* stream);
/* relu_src (may be NULL): the layer's input when that input is itself a ReLU output; the epilogue
 * then writes dX[:, :relu_cols] * (relu_src > 0), i.e. the dZ of the layer below (fused mask). */
/* dW[n_out, k] += dZ^T X, db += column sums of dZ (dZ = dY * act'(Y) supplied by the caller).
 * dW^T accumulates in registers across each CTA's row tiles, flushed once with atomics (csrc/wgrad_mn.cu).
 * Needs 16-byte aligned rows (ldx, lddz multiples of 4); k <= 256, n_out <= 128. */
int emer_linear_tc_bwd_weight(const float* x, int64_t ldx, const float* dz, int64_t lddz, float* dw,
                              float* db, int64_t n, int k, int n_out, void* stream);

/* ---- inverse-CDF resampling (replaces nerfacc.pdf.importance_sampling + _transform_stot,
 *      third_party/nerfacc_prop_net.py:153-160,172-175,299-339) ---------------------------- */
enum { EMER_STOT_UNIFORM = 0, EMER_STOT_LINDISP = 1, EMER_STOT_SQRT = 2, EMER_STOT_LOG = 3,
       EMER_STOT_UNIFORM_LINDISP = 4, EMER_STOT_UNIFORM_LINDISP_0 = 5 };
/* vals, cdfs: [R, m1]; out_s, out_t: [R, n+1]; out_bins (int32 [R, n+1], may be NULL) = the
 * upper-bound index p of each output edge.  bias: [R] stratified jitter in [0,1) or NULL (0.5).
 * s_min/s_max are the fp32 contract_fn(near/far) values computed by the caller. */
int emer_pdf_resample(const float* vals, const float* cdfs, int m1, int n, const float* bias,
                      float s_min, float s_max, int stot_kind, float* out_s, float* out_t,
                      int32_t* out_bins, int64_t n_rays, void* stream);

/* One whole proposal level in one launch (no-grad path of PropNetEstimator.sampling,
 * third_party/nerfacc_prop_net.py:147-170 + render_utils.py:314-324 + radiance_field.py:825-841):
 * resample n intervals from (prev_s, prev_cdf)[R, m1], s->t warp, march, contraction + selector, 3-D hash
 * grid, Linear(LF,64)-ReLU-Linear(64,1), trunc_exp(x-1), transmittance scan -> out_cdf[R, n+1].
 * out_s / out_t [R, n+1] are bit-identical to emer_pdf_resample's.  out_sigma [R, n] (may be NULL) keeps the level's
 * densities for emer_prop_level_bwd. */
int emer_prop_level(const emer_grid_desc* g, const float* prev_s, const float* prev_cdf, int m1, int n,
                    const float* bias, float s_min, float s_max, int stot_kind, const float* origins,
                    const float* dirs, const float* aabb6, int unbounded, const float* table,
                    const float* w0, const float* b0, const float* w1, const float* b1, float* out_s,
                    float* out_t, float* out_cdf, float* out_sigma, int64_t n_rays, void* stream);

/* Backward of one proposal level on the steps that update the proposal networks (the autograd graph the reference
 * builds through third_party/nerfacc_prop_net.py:161-170 -> render_utils.py:314-324 -> radiance_field.py:825-841 ->
 * nerfacc render_transmittance_from_density): the interlevel loss reaches the level only through d_cdf [R, n+1].
 * t_edges [R, n+1] and sigma [R, n] are the forward's out_t / out_sigma.  Recomputes positions, grid features and
 * hidden units; ACCUMULATES d_w0 [64, LF], d_b0 [64], d_w1 [64], d_b1 [1]; WRITES xc [R n, 3] (grid coordinates) and
 * d_enc [R n, LF], which emer_grid_bwd(g, xc, table, d_enc, d_table, NULL, R n) scatters into the table gradient.
 * Grids of 4 or 8 levels x 1 feature (the shipped proposal grids). */
int emer_prop_level_bwd(const emer_grid_desc* g, const float* t_edges, const float* sigma, const float* d_cdf, int n,
                        const float* origins, const float* dirs, const float* aabb6, int unbounded,
                        const float* table, const float* w0, const float* b0, const float* w1, float* xc,
                        float* d_enc, float* d_w0, float* d_b0, float* d_w1, float* d_b1, int64_t n_rays,
                        void* stream);

/* ---- anti-aliased interlevel loss of one proposal level, value and gradient in one launch (replaces, per level,
 *      the ~40 torch launches of PropNetEstimator.compute_loss, third_party/nerfacc_prop_net.py:182-240 with
 *      blur_stepfun :22-34 and sorted_interp_quad :37-60, and autograd's backward of them) -------------------------
 * s, cdf: [R, m] final-level edges (normalised) and CDF (a constant of the loss); prop_s, prop_cdf: [R, n1] of the
 * level; pulse_width: the level's blur radius.  ACCUMULATES sum_{rays, k} max(dq_k - dP_k, 0)^2 / (dP_k + 1e-5) into
 * loss_sum[0] (the reference's .mean() divides by R (n1 - 1)) and WRITES its gradient w.r.t. prop_cdf into
 * d_prop_cdf [R, n1] (may be NULL).  m <= 129, n1 <= 257. */
int emer_interlevel_loss(const float* s, const float* cdf, int m, const float* prop_s, const float* prop_cdf, int n1,
                         float pulse_width, float* loss_sum, float* d_prop_cdf, int64_t n_rays, void* stream);

/* ---- field tail: between the base MLP and the colour head (radiance_field.py:417-422,622-647) ---
 * forward : out[n, 0:W4] = [feats[n, 0:G] | sinenc((dir[ray]+1)/2) (33) | emb[idx[ray]] (E) | 0-pad], W4 = G+33+E
 *           rounded up to 4; ld_out (% 4 == 0, >= W4) is only the row stride, so the rows may sit inside a
 *           wider buffer (the colour head's skip-concatenation buffer) and no copy is needed later
 *           sigma[n] = exp(feats[n, 0] - 1)     (may be NULL);  n = ray * n_samples + sample
 * backward: d_out[:, 0] += d_sigma * exp(min(feats0 - 1, 15)) in place (so d_out[:, 0:G] IS d_feats);
 *           d_emb[idx[ray], :] += sum_s d_out[ray, s, G+33 : G+33+E]  (atomics, caller zeroes; may be NULL) */
int emer_field_tail_fwd(const float* feats, int64_t ld_feats, int g_dim, const float* dirs,
                        const int64_t* idx, const float* emb, int e_dim, float* out, int64_t ld_out,
                        float* sigma, int64_t n_rays, int n_samples, void* stream);
int emer_field_tail_bwd(const float* feats, int64_t ld_feats, float* d_out, int64_t ld_out, int g_dim,
                        const float* d_sigma, const int64_t* idx, float* d_emb, int e_dim, int64_t n_rays,
                        int n_samples, void* stream);

/* ---- the fused field chain (csrc/field_fused.cu): base MLP -> density + colour head in ONE wgmma kernel with the
 *      activations in registers.  Replaces the chain of nn.Linear / torch.cat / trunc_exp / sigmoid calls of
 *      radiance_fields/radiance_field.py:74-80,314-318 (base_mlp), :422 (density), :131-143,622-658 (query_rgb) and
 *      radiance_fields/mlp.py:38-46 for one block of hash-grid features.
 *   enc[N, k_enc] (k_enc = 32, 40 or 64; rows 32-byte aligned: ld_enc % 8 == 0, and so must be the save
 *   buffers)
 *   feats = relu(enc wb0^T + bb0) wb1^T + bb1        wb0 [64, k_enc], wb1 [n_feat, 64], n_feat = 64 | 128
 *   sigma[n] = exp(feats[n, 0] - 1)
 *   h0 = relu(geo w0g^T + ray_bias[ray, 0:64]),  h1 = relu(h0 w1h^T + geo w1g^T + ray_bias[ray, 64:128]),
 *   rgb[n, 0:3] = sigmoid(h1 w2^T + b2)              geo = feats[:, 0:64], ray = n / samples
 *   w0g / w1h / w1g are [64, 64] column blocks of the colour head's [64, 113] / [64, 177] weights (row strides ld_w0 /
 *   ld_w1); the per-ray input columns (direction encoding, appearance embedding) and the two layer biases arrive folded
 *   into ray_bias[R, 128] by the caller.
 *   save_hb [N,64] = relu(.) of the base layer, save_hg [N,128] = [h0 | geo], save_h1 [N,64], save_sem [N,64] =
 *   feats[:, 64:128]: what the backward pass needs; each may be NULL (inference), save_sem is required when
 *   n_feat == 128. */
int emer_field_fwd(const float* enc, int64_t ld_enc, int k_enc, const float* wb0, const float* bb0,
                   const float* wb1, const float* bb1, int n_feat, const float* w0g, int64_t ld_w0,
                   const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, const float* b2,
                   const float* ray_bias, int samples, float* sigma, float* rgb, float* save_hb, float* save_hg,
                   float* save_h1, float* save_sem, int64_t n, void* stream);

/* Backward of emer_field_fwd, data path (the autograd graph of the same reference lines), one kernel, every
 * intermediate gradient in registers:
 *   dz2[N,3] = d_rgb * rgb (1 - rgb);  dz1[N,64] = (dz2 w2) * (h1 > 0);
 *   d1[N,128] = [dz0 | dF]: dz0 = (dz1 w1h) * (h0 > 0), dF = dz1 w1g + dz0 w0g + d_geo, dF[:,0] += d_sigma * min(sigma, e^15)
 *   dzb[N,64] = (dF wb1[:64] + d_sem wb1[64:]) * (hb > 0);  d_enc[N, k_enc] = dzb wb0   (row stride ld_denc)
 *   d_ray_bias[R,128] += per-ray sums of [dz0 | dz1]   (caller zeroes; needs samples % 32 == 0; may be NULL)
 * hb / hg / h1 / rgb / sigma are emer_field_fwd's saves and outputs.  d_rgb, d_sigma, d_geo, d_sem, d_enc, dz2 may be
 * NULL; without d_rgb, dz2 is not written.  Row buffers 32-byte aligned, ld_denc % 8 == 0.  The weight gradients are X^T dZ products over dz2 / dz1 / d1 /
 * dzb (emer_field_wgrad). */
int emer_field_bwd(const float* d_rgb, const float* rgb, const float* d_sigma, const float* sigma,
                   const float* d_geo, const float* d_sem, const float* hb, const float* hg, const float* h1,
                   const float* wb0, int k_enc, const float* wb1, int n_feat, const float* w0g, int64_t ld_w0,
                   const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, float* dz2, float* dz1,
                   float* d1, float* dzb, float* d_enc, int64_t ld_denc, float* d_ray_bias, int samples,
                   int64_t n, void* stream);

/* Weight gradients of the fused field chain from emer_field_bwd's buffers, in one launch that reads every row buffer
 * once (csrc/field_wgrad.cu).  All outputs accumulate (+=; the caller zeroes):
 *   dwb0 [64, k_enc] += dzb^T enc,                 dbb0 [64]     += column sums of dzb
 *   dwb1 [n_feat, 64] += [dF | d_sem]^T hb,         dbb1 [n_feat] += column sums of [dF | d_sem]
 *   dw0g [64, 64] (row stride ld_w0) += dZ0^T geo
 *   dw1h, dw1g [64, 64] (row stride ld_w1) += dz1^T h0, dz1^T geo
 *   dw2 [3, 64] += dz2^T h1,                        db2 [3]       += column sums of dz2
 * with hg = [h0 | geo] [N,128] and d1 = [dZ0 | dF] [N,128].  enc [N, k_enc] has row stride ld_enc (% 4 == 0);
 * hb, h1, dz1, dzb, d_sem [N,64] and dz2 [N,3] are dense.  d_sem (n_feat = 128 only) may be NULL: dWb1's rows 64.. and
 * dbb1[64:] are then left as they are.  dz2 NULL (no colour gradient): only dwb0 / dbb0 / dwb1 / dbb1 are computed,
 * and hg, h1, dz1 and the head's outputs may be NULL.  Row buffers 16-byte aligned. */
int emer_field_wgrad(const float* enc, int64_t ld_enc, int k_enc, const float* hb, const float* hg, const float* h1,
                     const float* dz2, const float* dz1, const float* d1, const float* dzb, const float* d_sem,
                     int n_feat, float* dwb0, float* dbb0, float* dwb1, float* dbb1, float* dw0g, int64_t ld_w0,
                     float* dw1h, float* dw1g, int64_t ld_w1, float* dw2, float* db2, int64_t n, void* stream);

/* ---- volume rendering along rays (replaces nerfacc.render_transmittance_from_density /
 *      render_weight_from_density / accumulate_along_rays and the torch cumsum/searchsorted of
 *      radiance_fields/render_utils.py:73-115) ---------------------------------------------- */
/* per ray, S samples: weights, trans [R,S]; opacity (clamped to [1e-6,1]), depth, median_depth [R];
 * cdf_or_null [R, S+1] = 1 - cat(trans, 0) (nerfacc_prop_net.py:165-168). */
int emer_composite_fwd(const float* t0, const float* t1, const float* sigma, float* weights,
                       float* trans, float* opacity, float* depth, float* median_depth,
                       float* cdf, int64_t n_rays, int n_samples, void* stream);
/* dsigma[R,S] from any of g_weights, g_trans [R,S], g_opacity, g_depth [R] (NULL = zero). */
int emer_composite_bwd(const float* t0, const float* t1, const float* sigma, const float* weights,
                       const float* trans, const float* g_weights, const float* g_trans,
                       const float* g_opacity, const float* g_depth, float* dsigma,
                       int64_t n_rays, int n_samples, void* stream);
/* out[R, C] = sum_s w[R,S] * v[R,S,C] */
int emer_accumulate_fwd(const float* w, const float* v, float* out, int64_t n_rays, int n_samples,
                        int c, void* stream);
/* dw[R,S] (may be NULL) = sum_c g[R,C] v[R,S,C];  dv[R,S,C] (may be NULL) = w * g */
int emer_accumulate_bwd(const float* w, const float* v, const float* g, float* dw, float* dv,
                        int64_t n_rays, int n_samples, int c, void* stream);

/* ---- ray generation (replaces datasets/base/pixel_source.py:39-76 get_rays and the per-ray gathers / coordinate
 *      assembly of get_train_rays, :699-719) ------------------------------------------------------------------ */
/* Per ray i: m = img_idx[i] (or i when per_ray_mats, or 0), c2w[m] (4x4 row-major), intrinsics[m] (3x3):
 *   origins[i] = c2w[:3,3];  viewdirs[i] = R cam / (|R cam| + 1e-8), cam = ((x-cx+.5)/fx, (y-cy+.5)/fy, 1);
 *   norms[i] = |R cam|;  pixel_coords[i] = (y / height, x / width);  out_times[i] = timestamps[m].
 * img_idx (int64), norms, pixel_coords, out_times / timestamps may be NULL. */
int emer_gen_rays(const int64_t* img_idx, const float* x, const float* y, const float* c2w, const float* intrinsics,
                  int per_ray_mats, const float* timestamps, int height, int width, float* origins, float* viewdirs,
                  float* norms, float* pixel_coords, float* out_times, int64_t n, void* stream);

/* ---- optimizer (replaces torch.optim.Adam's step + optimizer.zero_grad() + tiny-cuda-nn's gradient memset,
 *      builders.py:50-61,114-120; train_emernerf.py:742-745,823-826) --------------------------------------------- */
/* One parameter block: n fp32 values of a parameter, its gradient and Adam moments (16-byte aligned, device). */
typedef struct emer_adam_block {
    float* param;
    float* grad;
    float* exp_avg;
    float* exp_avg_sq;
    int64_t n;
} emer_adam_block;
/* Adam (amsgrad = False) over n_blocks blocks in ONE launch; the consumed gradient is zeroed when zero_grad != 0.
 * blocks / prefix are DEVICE arrays: block b covers the virtual index range [prefix[b], prefix[b+1]) (prefix[b]
 * multiples of 4, prefix[n_blocks] = total).  hyper = device {step (already incremented), lr}: read at run time so
 * that a captured CUDA graph replays with the live values. */
int emer_adam_step(const emer_adam_block* blocks, const int64_t* prefix, int n_blocks, int64_t total,
                   const float* hyper, float beta1, float beta2, float eps, float weight_decay, int zero_grad,
                   void* stream);

/* ---- training losses (replaces the op-by-op torch of loss/base.py: RealValueLoss :83-146, SkyLoss :149-185,
 *      DepthLoss :188-269, LineOfSightLoss :272-335 with compute_line_of_sight_loss :430-464,
 *      DynamicRegularizationLoss :338-410), csrc/losses.cu ------------------------------------------------------------
 * Forward: ONE launch, no host sync.  out [2] (caller-owned, per call) receives out[0] = the loss value and out[1] = the
 * count its mean divides by (elements, valid rays, or rays with gt > 0), which the backward reads.  workspace: at least
 * EMER_LOSS_WORKSPACE_BYTES of device memory, zeroed once by its owner; the kernel leaves it zeroed again, so it is
 * reused by every call (and every CUDA-graph replay) on one stream -- calls that may run concurrently need separate
 * workspaces.  Sums are per CTA, then over CTAs in a fixed order (no float atomics): bit-identical on one device.
 * Backward: ONE launch; g is the upstream gradient (a device scalar); the gradients are WRITTEN (not accumulated).
 * pre: per-element factor before the mean; post: factor after it (the loss's coef). */
#define EMER_LOSS_WORKSPACE_BYTES 16384
enum {
    EMER_LOSS_L1 = 0, EMER_LOSS_L2 = 1, EMER_LOSS_SMOOTH_L1 = 2,    /* a = pred, b = target [n]; mean over n        */
    EMER_LOSS_DEPTH_L1 = 3, EMER_LOSS_DEPTH_L2 = 4,                 /* a = pred, b = gt depth [n]; p0 = max depth:  */
    EMER_LOSS_DEPTH_SMOOTH_L1 = 5,                                  /*   clamp(d / p0, 0, 1), mean over 0.01 < gt < p0 */
    EMER_LOSS_SKY_BCE = 6,                                          /* a = opacity, b = sky mask: BCE(a, 1 - b)     */
    EMER_LOSS_SPARSITY = 7,                                         /* a = density (b unused): mean(a)              */
    EMER_LOSS_ENTROPY = 8                                           /* a = dynamic, b = static density; p0 = skewness
                                                                       k, p1 = k - 1; da and/or db                  */
};
int emer_pointwise_loss_fwd(int kind, const float* a, const float* b, int64_t n, float p0, float p1, float pre,
                            float post, float* out, void* workspace, void* stream);
int emer_pointwise_loss_bwd(int kind, const float* a, const float* b, int64_t n, float p0, float p1, float pre,
                            float post, const float* fwd_out, const float* g, float* da, float* db, void* stream);

/* Per-ray sums over the S samples of [R, S] rows.
 *   LINE_OF_SIGHT: w = weights, t = t_vals [R, S], gt = gt depth [R]; eps, two_sigma_sq = 2 (eps/3)^2,
 *                  amp = 1 / sqrt(2 pi (eps/3)^2):  post * mean_r(pre * (mean_r empty_r + mean_r near_r) * [gt_r > 0])
 *   SKY_WEIGHTS:   w = weights, t unused, gt = sky mask [R]:  post * mean_r(sum_s w^2 * sky_r)
 *   SIGHT:         as LINE_OF_SIGHT without the ray mask and its mean: post * pre * (mean_r empty_r + mean_r near_r)
 * dw [R, S] is d loss / d w. */
enum { EMER_RAY_LOSS_LINE_OF_SIGHT = 0, EMER_RAY_LOSS_SKY_WEIGHTS = 1, EMER_RAY_LOSS_SIGHT = 2 };
int emer_ray_loss_fwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays, int n_samples, float eps,
                      float two_sigma_sq, float amp, float pre, float post, float* out, void* workspace, void* stream);
int emer_ray_loss_bwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays, int n_samples, float eps,
                      float two_sigma_sq, float amp, float pre, float post, const float* fwd_out, const float* g,
                      float* dw, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EMER_B200_H */
