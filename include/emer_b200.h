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

/* The flow variants' dynamic branch on the same chain (csrc/field_fused.cu, the kernels above with three queries per
 * row).  enc holds 3N rows: rows [0, N) the current encodings, [N, 2N) the forward-warped and [2N, 3N) the
 * backward-warped ones.  Each goes through the base MLP, and the features blend before the density and the colour head
 * (radiance_field.py:449-460, the same operation order):
 *   F_q = relu(enc_q wb0^T + bb0) wb1^T + bb1,  feats = (F_c + 0.5 F_f + 0.5 F_b) / 2;  sigma, rgb as emer_field_fwd.
 * save_hb is [3N, 64]; save_hg [N, 128] (required: its geometry half carries the blend) and save_sem [N, 64] hold the
 * blended features.  rgb == NULL: density only (the lidar pass); the colour head is skipped and ray_bias, save_h1 may be
 * NULL. */
int emer_flow_field_fwd(const float* enc, int64_t ld_enc, int k_enc, const float* wb0, const float* bb0,
                        const float* wb1, const float* bb1, int n_feat, const float* w0g, int64_t ld_w0,
                        const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, const float* b2,
                        const float* ray_bias, int samples, float* sigma, float* rgb, float* save_hb, float* save_hg,
                        float* save_h1, float* save_sem, int64_t n, void* stream);

/* Backward of emer_flow_field_fwd: emer_field_bwd's data path for the blended features, whose gradient dF fans out to the
 * three queries as dF / 2, dF / 4, dF / 4.  d1 is [3N, 128]: rows [0, N) = [dz0 | dF_c], rows N.. = [unused | dF_q];
 * dzb and d_enc (row stride ld_denc) hold 3N rows, d_sem_q [3N, 64] the three queries' d_sem (required with d_sem).  The
 * base MLP's weight gradients are emer_field_wgrad over the 3N rows (the colour head's over the first N);
 * h1 == NULL: density only (no d_rgb, dz2, d_ray_bias). */
int emer_flow_field_bwd(const float* d_rgb, const float* rgb, const float* d_sigma, const float* sigma,
                        const float* d_geo, const float* d_sem, const float* hb, const float* hg, const float* h1,
                        const float* wb0, int k_enc, const float* wb1, int n_feat, const float* w0g, int64_t ld_w0,
                        const float* w1h, const float* w1g, int64_t ld_w1, const float* w2, float* dz2, float* dz1,
                        float* d1, float* dzb, float* d_enc, int64_t ld_denc, float* d_ray_bias, float* d_sem_q,
                        int samples, int64_t n, void* stream);

/* The flow warp of the temporal aggregation (csrc/flow_branch.cu; radiance_field.py:449-452), both directions in one
 * launch.  pos [N,3], flow [N,6] = [forward | backward], noise [N] (row stride ld_noise; NULL: 1, the eval renders),
 * t [N], time_diff: one float on the device (the model's time step may be a device tensor; reading it on the host would
 * stall the stream).  coords [2N,4] (16-byte aligned): row i = [contract(pos + flow[:,0:3] noise) | clamp(t + time_diff noise, 0, 1)],
 * row N + i = [contract(pos + flow[:,3:6] noise) | clamp(t - time_diff noise, 0, 1)], with the in-cube selector. */
int emer_flow_warp_fwd(const float* pos, const float* flow, const float* noise, int64_t ld_noise, const float* t,
                       const float* aabb6, const float* time_diff, int unbounded, float* coords, int64_t n, void* stream);

/* Backward of emer_flow_warp_fwd: d_flow [N,6] (written) from d_coords [2N,4] (the grid input gradient of those rows;
 * the time column is ignored) through the contraction's Jacobian, the selector and noise. */
int emer_flow_warp_bwd(const float* pos, const float* flow, const float* noise, int64_t ld_noise, const float* aabb6,
                       int unbounded, const float* d_coords, float* d_flow, int64_t n, void* stream);

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

/* ---- the whole body of `rendering` in one launch each way (replaces radiance_fields/render_utils.py:48-287: the
 *      static / dynamic ratios, the shadow product, the blended colour and features, every accumulate_along_rays, the
 *      sky and PE terms and the decomposition outputs), csrc/render.cu ---------------------------------------------
 * Per ray, S samples, C feature channels (1 <= C <= 256).  Every input but t0, t1, sigma may be NULL (absent); every
 * output may be NULL (not wanted).  Per-sample tensors are [R,S] or [R,S,3] / [R,S,C] rows, per-ray ones [R], [R,3] or
 * [R,C], all dense, except the flows: R*S rows of 3 floats with row stride ld_flow (column slices of the flow MLP's
 * 6-wide rows).  w = weights, r_s = sigma_s / (sigma + 1e-6), r_d = sigma_d / (sigma + 1e-6), w_s / w_d = the weights
 * of sigma_s / sigma_d alone, op = opacity:
 *   weights, trans, opacity, depth, median_depth      bit-identical to emer_composite_fwd's
 *   rgb           = sum w*rgb  (rgb given)  or  sum w*(r_s*rgb_s*(1 - shadow) + r_d*rgb_d),  + rgb_sky*(1 - op)
 *   shadow_ratio  = sum w*shadow^2
 *   dino_pe_free  = sum w*dino  or  sum w*(r_s*dino_s + r_d*dino_d),  + dino_sky*(1 - op);   dino = dino_pe_free + dino_pe
 * and, for evaluation (emer_render_bwd has no gradient for these):
 *   static_ / dynamic_opacity, _depth                  as opacity / depth of sigma_s / sigma_d
 *   static_rgb    = sum w_s*rgb_s + rgb_sky*(1 - static_opacity);   dynamic_rgb = sum w_d*rgb_d
 *   shadow_reduced_static_rgb = sum w_s*rgb_s*(1 - shadow);  shadow_only_static_rgb = sum w_s*rgb_s*shadow + 1 - shadow
 *   shadow        = sum w*shadow;   forward_flow / backward_flow = sum w_d*flow
 *   static_dino   = sum w_s*dino_s + dino_sky*(1 - op)  (the TOTAL opacity, as the reference);  dynamic_dino = sum w_d*dino_d */
typedef struct emer_render_in {
    const float* t0;            /* [R,S] */
    const float* t1;            /* [R,S] */
    const float* sigma;         /* [R,S] */
    const float* sigma_s;       /* [R,S]; sigma_s and sigma_d come together */
    const float* sigma_d;
    const float* rgb;           /* [R,S,3] */
    const float* rgb_s;         /* [R,S,3]; rgb_s and rgb_d (and the sigmas) come together */
    const float* rgb_d;
    const float* shadow;        /* [R,S] */
    const float* rgb_sky;       /* [R,3] */
    const float* dino;          /* [R,S,C] */
    const float* dino_s;        /* [R,S,C]; dino_s and dino_d (and the sigmas) come together */
    const float* dino_d;
    const float* dino_sky;      /* [R,C] */
    const float* dino_pe;       /* [R,C] */
    const float* fwd_flow;      /* R*S rows of 3, row stride ld_flow */
    const float* bwd_flow;
    int64_t ld_flow;
    int64_t n_rays;
    int32_t n_samples;
    int32_t n_dino;             /* C */
} emer_render_in;

typedef struct emer_render_out {
    float* weights;             /* [R,S] */
    float* trans;               /* [R,S] */
    float* opacity;             /* [R] */
    float* depth;
    float* median_depth;
    float* rgb;                 /* [R,3] */
    float* shadow_ratio;        /* [R] */
    float* dino;                /* [R,C] */
    float* dino_pe_free;        /* [R,C] */
    float* static_opacity;      /* [R] */
    float* dynamic_opacity;
    float* static_depth;
    float* dynamic_depth;
    float* static_rgb;          /* [R,3] */
    float* dynamic_rgb;
    float* shadow_reduced_static_rgb;
    float* shadow_only_static_rgb;
    float* shadow;              /* [R] */
    float* forward_flow;        /* [R,3] */
    float* backward_flow;
    float* static_dino;         /* [R,C] */
    float* dynamic_dino;
} emer_render_out;

/* Gradients of emer_render_fwd's training outputs (NULL = zero) and of its inputs (WRITTEN, not accumulated; NULL =
 * not wanted).  Deterministic: no float atomics. */
typedef struct emer_render_grad {
    const float* g_weights;     /* [R,S]: the line-of-sight and sky-weight losses differentiate the weights */
    const float* g_trans;       /* [R,S] */
    const float* g_opacity;     /* [R] */
    const float* g_depth;
    const float* g_rgb;         /* [R,3] */
    const float* g_shadow_ratio;/* [R] */
    const float* g_dino;        /* [R,C] */
    const float* g_dino_pe_free;/* [R,C] */
    float* d_sigma;             /* [R,S] */
    float* d_sigma_s;
    float* d_sigma_d;
    float* d_rgb;               /* [R,S,3] */
    float* d_rgb_s;
    float* d_rgb_d;
    float* d_shadow;            /* [R,S] */
    float* d_rgb_sky;           /* [R,3] */
    float* d_dino;              /* [R,S,C] */
    float* d_dino_s;
    float* d_dino_d;
    float* d_dino_sky;          /* [R,C] */
    float* d_dino_pe;
} emer_render_grad;

int emer_render_fwd(const emer_render_in* in, const emer_render_out* out, void* stream);
/* weights, trans: emer_render_fwd's outputs for the same inputs. */
int emer_render_bwd(const emer_render_in* in, const float* weights, const float* trans, const emer_render_grad* grad,
                    void* stream);

/* ---- ray generation (replaces datasets/base/pixel_source.py:39-76 get_rays and the per-ray gathers / coordinate
 *      assembly of get_train_rays, :699-719) ------------------------------------------------------------------ */
/* Per ray i: m = img_idx[i] (or i when per_ray_mats, or 0), c2w[m] (4x4 row-major), intrinsics[m] (3x3):
 *   origins[i] = c2w[:3,3];  viewdirs[i] = R cam / (|R cam| + 1e-8), cam = ((x-cx+.5)/fx, (y-cy+.5)/fy, 1);
 *   norms[i] = |R cam|;  pixel_coords[i] = (y / height, x / width);  out_times[i] = timestamps[m].
 * img_idx (int64), norms, pixel_coords, out_times / timestamps may be NULL. */
int emer_gen_rays(const int64_t* img_idx, const float* x, const float* y, const float* c2w, const float* intrinsics,
                  int per_ray_mats, const float* timestamps, int height, int width, float* origins, float* viewdirs,
                  float* norms, float* pixel_coords, float* out_times, int64_t n, void* stream);

/* ---- training batches of pixel rays (replaces ScenePixelSource.get_train_rays with its samplers,
 *      datasets/base/pixel_source.py:564-731) ------------------------------------------------------------------ */
/* workspace: at least EMER_RAYBATCH_WORKSPACE_BYTES of device memory, zeroed once by its owner and left zeroed by
 * every call (as the loss workspace below), so it is reused by every call and graph replay on one stream. */
#define EMER_TOPK_MAX_K 16384
#define EMER_RAYBATCH_WORKSPACE_BYTES 141376
/* The selection of torch.multinomial(p[cand].reshape(-1), k, replacement=False) = topk(p[cand] / q, k) for a caller-
 * drawn q ~ Exp(1): out_idx (int64 [k]) gets the j in [0, M = n_cand * plane) of the k largest
 * p[cand[j / plane] * plane + j % plane] / q[j] (IEEE division), by descending key, then ascending j.  p: the error
 * maps [N, plane] (fp32, dense), cand: int64 [n_cand] image indices, q: fp32 [M].  The keys must be finite or +inf and
 * non-negative (the caller validates p as torch.multinomial does).  1 <= k <= min(EMER_TOPK_MAX_K, M), M < 2^31.
 * Five launches: three radix-select passes and a collection over the keys, and a one-CTA sort of the k survivors. */
int emer_topk_ratio(const float* p, int64_t plane, const int64_t* cand, int64_t n_cand, const float* q, int64_t k,
                    int64_t* out_idx, void* workspace, void* stream);

#define EMER_PIXEL_BATCH_MAX_FEATURES 256
/* Inputs of a training batch: n_uniform rays from the uniform draws, then n_importance rays from the selected indices.
 * Images are [n_images, height, width] (rgb with 3 channels), features [n_images, feat_h, feat_w, feat_c]; every
 * table is dense and on the device; images, masks, features, timestamps and cam_ids may be NULL. */
typedef struct EmerPixelBatchIn {
    const int64_t* cand;                      /* [n_cand] image indices the draws refer to                           */
    const int64_t* u_pick;                    /* [n_uniform] positions in cand                                      */
    const int64_t* u_x;                       /* [n_uniform] pixel columns                                          */
    const int64_t* u_y;                       /* [n_uniform] pixel rows                                             */
    const int64_t* i_sel;                     /* [n_importance] j of emer_topk_ratio over the maps [cand, map_h, map_w] */
    const int64_t* i_dy;                      /* [n_importance] row offsets in [0, map_downscale)                   */
    const int64_t* i_dx;                      /* [n_importance] column offsets                                      */
    const float* images;                      /* [N, H, W, 3]                                                       */
    const float* sky_masks;                   /* [N, H, W]                                                          */
    const float* dynamic_masks;               /* [N, H, W]                                                          */
    const float* features;                    /* [N, feat_h, feat_w, feat_c]                                        */
    const float* timestamps;                  /* [N]                                                                */
    const int64_t* cam_ids;                   /* [N]                                                                */
    const float* c2w;                         /* [N, 4, 4]                                                          */
    const float* intrinsics;                  /* [N, 3, 3]                                                          */
    int64_t n_uniform, n_importance;
    int32_t height, width;
    int32_t map_h, map_w, map_downscale;
    int32_t feat_h, feat_w, feat_c;
    float feat_scale_y, feat_scale_x;         /* feature row = (int)((float)y * feat_scale_y), likewise the column  */
} EmerPixelBatchIn;

/* Outputs, [R = n_uniform + n_importance] rows; an output whose input is NULL must be NULL. */
typedef struct EmerPixelBatchOut {
    int64_t* img_idx;                         /* [R]                                                                */
    int64_t* cam_idx;                         /* [R] cam_ids[img]                                                   */
    float* pixels;                            /* [R, 3]                                                             */
    float* sky_masks;                         /* [R]                                                                */
    float* dynamic_masks;                     /* [R]                                                                */
    float* features;                          /* [R, feat_c]                                                        */
    float* timestamps;                        /* [R] timestamps[img]                                                */
    float* origins;                           /* [R, 3]                                                             */
    float* viewdirs;                          /* [R, 3]                                                             */
    float* norms;                             /* [R, 1]                                                             */
    float* pixel_coords;                      /* [R, 2] (y * (1/height), x * (1/width)), as torch computes y / H on CUDA */
} EmerPixelBatchOut;

/* One launch: for uniform ray i, img = cand[u_pick[i]], (y, x) = (u_y[i], u_x[i]); for importance ray t,
 * (c, row, col) = idx_to_3d(i_sel[t]), img = cand[c], y = clamp(row * map_downscale + i_dy[t], 0, height - 1), x
 * likewise; then the gathers and the ray of emer_gen_rays at (x, y) with img's camera. */
int emer_pixel_batch(const EmerPixelBatchIn* in, const EmerPixelBatchOut* out, void* stream);

/* ---- whole-image render rays and the pixel error map (csrc/errormap.cu; replaces ScenePixelSource.get_render_rays,
 *      datasets/base/pixel_source.py:733-846, without the resize of the image, and update_pixel_error_maps, :491-517,
 *      with the host copies of radiance_fields/video_utils.py:104-468 that feed it) ---------------------------------- */
/* Inputs of emer_image_rays: the source's tables at full size [N, height, width], as EmerPixelBatchIn; masks,
 * features, timestamps and cam_ids may be NULL. */
typedef struct EmerImageRaysIn {
    const float* sky_masks;                   /* [N, height, width]                                                 */
    const float* dynamic_masks;               /* [N, height, width]                                                 */
    const float* features;                    /* [N, feat_h, feat_w, feat_c]                                        */
    const float* timestamps;                  /* [N]                                                                */
    const int64_t* cam_ids;                   /* [N]                                                                */
    const float* c2w;                         /* [N, 4, 4]                                                          */
    const float* intrinsics;                  /* [N, 3, 3]                                                          */
    int64_t first_image, n_images;            /* the images [first_image, first_image + n_images)                   */
    int32_t height, width;                    /* full size                                                          */
    int32_t h, w;                             /* rendered size, the resized image's                                 */
    float downscale;                          /* the source's downscale_factor d, as fp32: K * d                    */
    float mask_scale_y, mask_scale_x;         /* nearest source row = min(floor(y * mask_scale_y), height - 1);     */
                                              /* (float)(1.0 / d), torch's scale for interpolate(scale_factor=d)    */
    int32_t feat_h, feat_w, feat_c;
    float feat_scale_y, feat_scale_x;         /* feature row = (int)((float)y * feat_scale_y): featmap_downscale / d */
} EmerImageRaysIn;

/* Outputs, [R = n_images * h * w] rows in (image, y, x) order; an output whose input is NULL must be NULL. */
typedef struct EmerImageRaysOut {
    float* origins;                           /* [R, 3]                                                             */
    float* viewdirs;                          /* [R, 3]                                                             */
    float* norms;                             /* [R, 1]                                                             */
    float* pixel_coords;                      /* [R, 2] (y * (1/h), x * (1/w)), as torch computes y / h on CUDA     */
    float* timestamps;                        /* [R] timestamps[img]                                                */
    int64_t* img_idx;                         /* [R]                                                                */
    int64_t* cam_idx;                         /* [R] cam_ids[img]                                                   */
    float* sky_masks;                         /* [R] the nearest source pixel                                       */
    float* dynamic_masks;                     /* [R]                                                                */
    float* features;                          /* [R, feat_c]                                                        */
} EmerImageRaysOut;

/* One launch: for every pixel (y, x) of the h x w grid of every image, the ray of emer_gen_rays with the intrinsics
 * scaled by d in fp32, the pixel coordinates, and the gathers of get_render_rays at the nearest-mode source pixel and
 * at get_features' cell. */
int emer_image_rays(const EmerImageRaysIn* in, const EmerImageRaysOut* out, void* stream);

/* ---- render rays of a camera that moves between two keyframe images (csrc/errormap.cu; the producer of
 *      raygen.CameraTrajectory's frames, a new-view counterpart of get_render_rays) -------------------------------- */
/* Inputs: the source's full-size tables, as EmerImageRaysIn; timestamps may be NULL. */
typedef struct EmerTrajectoryRaysIn {
    const float* c2w;                         /* [N, 4, 4]                                                          */
    const float* intrinsics;                  /* [N, 3, 3]                                                          */
    const float* timestamps;                  /* [N]                                                                */
    int64_t n_images;                         /* N                                                                  */
    int64_t image_a, image_b;                 /* the keyframes of the segment                                       */
    int64_t cam_id;                           /* written to cam_idx                                                 */
    double offset[3];                         /* added to the origin along the camera's own axes (columns of c2w)   */
    int32_t frac_num, frac_den;               /* the frame lies at f = frac_num / frac_den, 0 <= frac_num < frac_den */
    int32_t h, w;                             /* rendered size                                                      */
    float downscale;                          /* the source's downscale_factor d, as fp32: K * d                    */
} EmerTrajectoryRaysIn;

/* Outputs, [R = h * w] rows in (y, x) order; timestamps must be NULL when its input is, sky_masks may be NULL. */
typedef struct EmerTrajectoryRaysOut {
    float* origins;                           /* [R, 3]                                                             */
    float* viewdirs;                          /* [R, 3]                                                             */
    float* norms;                             /* [R, 1]                                                             */
    float* pixel_coords;                      /* [R, 2] (y * (1/h), x * (1/w)), as emer_image_rays                 */
    float* timestamps;                        /* [R] t_a + f (t_b - t_a) in fp32                                    */
    int64_t* img_idx;                         /* [R] image_a when 2 frac_num <= frac_den, else image_b              */
    int64_t* cam_idx;                         /* [R] cam_id                                                         */
    float* sky_masks;                         /* [R] zeros                                                          */
} EmerTrajectoryRaysOut;

/* One launch, no allocation.  The pose: keyframe a's c2w bit for bit when frac_num == 0; otherwise the slerp of the two
 * keyframes' rotations (as unit quaternions, q_b negated when q_a . q_b < 0; a normalised lerp when the dot exceeds
 * 0.9995) and the lerp of their origins, in fp64, rounded to fp32.  Then origin += R offset (fp64, rounded), R the
 * frame's rotation.  The intrinsics are keyframe a's times d.  Each pixel's ray and pixel coordinates are
 * emer_image_rays' with that pose, so a frame with frac_num == 0 and a zero offset equals emer_image_rays of
 * image a. */
int emer_trajectory_rays(const EmerTrajectoryRaysIn* in, const EmerTrajectoryRaysOut* out, void* stream);

/* workspace: at least EMER_ERRORMAP_WORKSPACE_BYTES of device memory, zeroed once by its owner and left zeroed by
 * emer_error_map_normalize (as the raybatch workspace above).  Between the two calls it holds the running minimum and
 * maximum of the map. */
#define EMER_ERRORMAP_WORKSPACE_BYTES 16
/* For n pixels (one or more whole images): map[i] = mean_c |gt[i, c] - rgb[i, c]| as torch computes it on the CPU
 * (((e0 + e1) + e2) / 3 in fp32), times 5 (fp32) where opacity[i] > 0.1f when opacity is not NULL.  gt and rgb are
 * [n, 3], opacity [n], map [n] (the images' rows of the map).  Folds the minimum and maximum into the workspace with
 * integer atomics on the fp32 bit patterns (the errors are >= 0, or NaN, which orders above them), so the result does
 * not depend on the order of the CTAs. */
int emer_error_map(const float* gt, const float* rgb, const float* opacity, int64_t n, float* map, void* workspace,
                   void* stream);
/* map[i] = (map[i] - min) / (max - min) over the n entries of the whole map, with the minimum and maximum every
 * emer_error_map call since the last normalisation folded in: fp32 subtractions and an IEEE division, as torch
 * computes them on CUDA with 0-d tensor operands.  A NaN error or a constant map gives NaN (0 / 0), as there.  Zeroes
 * the workspace. */
int emer_error_map_normalize(float* map, int64_t n, void* workspace, void* stream);

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
/* The same for LINE_OF_SIGHT and SIGHT, with the per-step constants read from device memory at kernel start:
 * consts [4] fp32 = {eps, two_sigma_sq, amp, pre}.  A CUDA graph that captures these calls replays with whatever the
 * caller last wrote there.  With the values the float entries receive, value and gradient are bit-identical to theirs. */
int emer_ray_loss_live_fwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays, int n_samples,
                           const float* consts, float post, float* out, void* workspace, void* stream);
int emer_ray_loss_live_bwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays, int n_samples,
                           const float* consts, float post, const float* fwd_out, const float* g, float* dw,
                           void* stream);

/* ---- the flow variants' cycle loss and flow statistics (replaces the inline block of train_emernerf.py:700-740)
 * f = forward_flow, b = backward_flow, fpb = forward_pred_backward_flow, bpf = backward_pred_forward_flow: each n rows
 * of 3 floats (n = R * S samples), row i at x + i * ld_x (ld_x >= 3: a column slice of a wider row is read in place).
 *   value = coef * (0.5 * mean((f + fpb)^2 + (b + bpf)^2)), the mean over all 3n elements
 * Forward: ONE launch, no host sync, n >= 1.  out [6] (caller-owned): out[0] = value, out[1] = 3n (the count the mean
 * divides by, read by the backward), out[2..5] = the maximum row norm of f, b, fpb, bpf (NaN if any row of that input
 * holds a NaN).  workspace as for the losses above.  The sum is per CTA, then over CTAs in a fixed order.
 * Backward: ONE launch; f and b are constants.  d_fpb, d_bpf: [n, 3] contiguous, WRITTEN; either may be NULL.
 *   d = 2 (f + fpb) * (g * coef * 0.5 / out[1])  (and likewise for b, bpf) */
int emer_cycle_loss_fwd(const float* f, int64_t ld_f, const float* b, int64_t ld_b, const float* fpb, int64_t ld_fpb,
                        const float* bpf, int64_t ld_bpf, int64_t n, float coef, float* out, void* workspace,
                        void* stream);
int emer_cycle_loss_bwd(const float* f, int64_t ld_f, const float* b, int64_t ld_b, const float* fpb, int64_t ld_fpb,
                        const float* bpf, int64_t ld_bpf, int64_t n, float coef, const float* fwd_out, const float* g,
                        float* d_fpb, float* d_bpf, void* stream);

/* ---- evaluation metrics (csrc/metrics.cu).  Each call is ONE launch with no host sync; results are fp64 in a
 *      caller-owned device array.  workspace: at least EMER_METRICS_WORKSPACE_BYTES of device memory, zeroed once by
 *      its owner and left zeroed by every call (as the loss workspace above); sums are per CTA, then over CTAs in a
 *      fixed order, so results are bit-identical on one device. --------------------------------------------------- */
#define EMER_METRICS_WORKSPACE_BYTES 81920
/* The metric block of one evaluation image (replaces radiance_fields/video_utils.py:205-247: compute_psnr, two
 * skimage.metrics.structural_similarity calls on host copies, the masked PSNRs by boolean indexing, and the feature
 * PSNRs).  pred, target: [H, W, C] dense, 1 <= C <= 4, H, W >= 7.  mask: [H, W] (nonzero = in the mask) or NULL.
 * feat_pred, feat_target: H*W rows of feat_channels (<= 256) floats with row strides ld_feat_*, or both NULL.
 * SSIM as skimage's (data_range 1, channel_axis -1): 7x7 uniform window with scipy's 'reflect' border, sample
 * covariance 49/48, C1 = 0.01^2, C2 = 0.03^2, moments in fp64; ssim = mean over the interior [3, H-3) x [3, W-3) of
 * every channel; masked_ssim = mean of the uncropped map over the masked pixels x C.  out[EMER_IMAGE_METRICS_OUT]:
 * PSNR = -10 log10(mean squared error); a metric without its inputs (no mask, empty mask, no features) is NaN, and
 * MASK_COUNT is NaN without a mask.  The extrema propagate NaN (as numpy's). */
enum {
    EMER_METRIC_PSNR = 0, EMER_METRIC_SSIM = 1, EMER_METRIC_MASKED_PSNR = 2, EMER_METRIC_MASKED_SSIM = 3,
    EMER_METRIC_FEAT_PSNR = 4, EMER_METRIC_MASKED_FEAT_PSNR = 5, EMER_METRIC_MASK_COUNT = 6,
    EMER_METRIC_PRED_MIN = 7, EMER_METRIC_PRED_MAX = 8, EMER_METRIC_TARGET_MIN = 9, EMER_METRIC_TARGET_MAX = 10,
    EMER_IMAGE_METRICS_OUT = 11
};
int emer_image_metrics(const float* pred, const float* target, int64_t height, int64_t width, int channels,
                       const float* mask, const float* feat_pred, int64_t ld_feat_pred, const float* feat_target,
                       int64_t ld_feat_target, int feat_channels, double* out, void* workspace, void* stream);
/* compute_valid_depth_rmse (datasets/metrics.py:12-28) without boolean indexing: over n values,
 * out[0] = sqrt(mean((p - t)^2 over t > 0)) (NaN when no t > 0), out[1] = that count, and from the same pass
 * out[2] = -10 log10(mean((p - t)^2) over all n), the PSNR of compute_psnr (datasets/metrics.py:31-47). */
int emer_depth_rmse(const float* pred, const float* target, int64_t n, double* out, void* workspace, void* stream);
/* compute_scene_flow_metrics (datasets/metrics.py:73-128) over n points of [n, 3] dense pred / labels:
 * out[0] = EPE3D, out[1] = acc3d_strict, out[2] = acc3d_relax, out[3] = outlier, out[4] = angle_error (NaN when no
 * |label| > 0.1), out[5] = the points in the angle mean, out[6] = n.  The fractions are counts / n; the dot products
 * are clamped to the fp32 value of +-(1 - 1e-7), as torch rounds the reference's bounds. */
int emer_scene_flow_metrics(const float* pred, const float* labels, int64_t n, double* out, void* workspace,
                            void* stream);
/* The lidar scene-flow evaluation of one chunk of a frame (replaces the per-frame body of the reference's flow
 * evaluation, train_emernerf.py:248-281: the boolean indexes on lidar_flow_class != -1 and on the ground, the
 * dynamic-density gate and compute_scene_flow_metrics with its host copies).  n points: pred rows of 3 floats with
 * row stride ld_pred (>= 3; the forward flow read in place from the field's [n, 6] flow output), dynamic_density [n],
 * labels [n, 3] dense, flow_class int64 [n], ground [n] (nonzero = ground) or NULL to keep the ground.  A point is
 * valid when flow_class != -1 and counted when it is valid and not ground.  Over the counted points, with
 * pred *= 0 where dynamic_density < threshold (NaN stays NaN, a negative value gives -0, a NaN density is not gated),
 * the terms of emer_scene_flow_metrics are ADDED into sums[EMER_LIDAR_FLOW_SUMS] (fp64): the EPE sum, the strict,
 * relaxed and outlier counts, the angle sum and the angle count (|label| > 0.1), then the counted and the valid points.
 * One launch, no host sync, so the chunks of a frame add into one row; the last CTA adds the per-CTA sums in CTA order,
 * so the row is bit-identical on one device.  With n = 0 the inputs may be NULL (an empty tensor's data).  workspace:
 * the metrics workspace above. */
enum {
    EMER_LIDAR_FLOW_EPE = 0, EMER_LIDAR_FLOW_STRICT = 1, EMER_LIDAR_FLOW_RELAX = 2, EMER_LIDAR_FLOW_OUTLIER = 3,
    EMER_LIDAR_FLOW_ANGLE = 4, EMER_LIDAR_FLOW_ANGLE_COUNT = 5, EMER_LIDAR_FLOW_COUNTED = 6, EMER_LIDAR_FLOW_VALID = 7,
    EMER_LIDAR_FLOW_SUMS = 8
};
int emer_lidar_flow_accumulate(const float* pred, int64_t ld_pred, const float* dynamic_density, const float* labels,
                               const int64_t* flow_class, const uint8_t* ground, int64_t n, float threshold,
                               double* sums, void* workspace, void* stream);

/* ---- few-shot occupancy evaluation (csrc/occupancy.cu; replaces datasets/metrics.py:249-472, collect_centroids and
 *      eval_few_shot_occ with knn_predict(knn_k=1, similarity="cosine"), and their boolean indexing, second field pass
 *      and per-class .item() calls).  n voxels: feat rows of `channels` floats with row stride ld_feat (channels a
 *      multiple of 4, at most EMER_OCC_MAX_CHANNELS; feat and ld_feat 16-byte aligned), density with stride
 *      ld_density, labels int64.  A voxel is measured when density > threshold (strict; NaN fails).  Both calls ADD
 *      into caller-owned buffers with one launch and no host sync, so frames and chunks accumulate.  workspace: at
 *      least EMER_OCC_WORKSPACE_BYTES of device memory, zeroed once by its owner and left zeroed by every call (as
 *      the metrics workspace above); per-CTA records are added in CTA order, so results are bit-identical on one
 *      device. -------------------------------------------------------------------------------------------------- */
#define EMER_OCC_MAX_CHANNELS 256
#define EMER_OCC_MAX_CLASSES 32
#define EMER_OCC_WORKSPACE_BYTES 16912640
/* For the measured voxels with 0 <= label < n_classes (n_classes <= 32): sums[label, :] += feat row (fp64
 * [n_classes, channels]) and counts[label] += 1 (int64 [n_classes]).  Other labels are skipped. */
int emer_occ_accumulate(const float* feat, int64_t ld_feat, int channels, const float* density, int64_t ld_density,
                        const int64_t* labels, int64_t n, int n_classes, float threshold, double* sums,
                        int64_t* counts, void* workspace, void* stream);
/* For the measured voxels: prediction = label_bank[argmax_j dot(q, c_j / (|c_j| + 1e-7))] in fp64 over the fp32
 * centroids [n_classes, channels] (dense) and label_bank int64 [n_classes]; an exact tie goes to the lowest j.
 * counts int64 [2 n_classes + 2] accumulates: [0, n_classes) voxels per label, [n_classes, 2 n_classes) correct
 * predictions per label, [2 n_classes] measured voxels, [2 n_classes + 1] measured voxels whose label is outside
 * [0, n_classes) (not classified). */
int emer_occ_classify(const float* feat, int64_t ld_feat, int channels, const float* density, int64_t ld_density,
                      const int64_t* labels, int64_t n, const float* centroids, int n_classes,
                      const int64_t* label_bank, float threshold, int64_t* counts, void* workspace, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* EMER_B200_H */
