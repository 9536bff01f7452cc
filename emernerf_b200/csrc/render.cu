// The body of `rendering` (radiance_fields/render_utils.py:48-287) in one launch each way: the transmittance scan,
// the static / dynamic ratios, the shadow product, the blended colour and features, every accumulate_along_rays, the
// sky and PE terms and the evaluation-only decomposition.  Replaces, for a dynamic / flow / flow_feat field, ~20 torch
// elementwise ops and 3-14 emer_accumulate_* launches per pass, each reading or writing an [N, 3..64] temporary.
//
// Layout as composite.cu: one warp per ray.  Per-sample scalars (sigma, weights, ratios, colour) are handled with
// lanes striding the samples; the [S, C] feature rows with lanes striding the channels, sample by sample, with the
// per-sample weight factors broadcast from the lane that owns the sample (so both kinds of row are read coalesced).
//
// Backward (no float atomics; every output element has one writer):
//   x_i = sigma_i*delta_i, T_i = exp(-sum_{j<i} x_j), w_i = T_i (1 - exp(-x_i)), op = clamp(sum w, 1e-6, 1)
//   F  = sum_i w_i v_dino_i + dino_sky (1 - op);  g_F = g_dino + g_dino_pe_free   (dino = F + dino_pe, dino_pe_free = F)
//   G_i = g_w_i + g_rgb.v_rgb_i + g_shr sh_i^2 + g_F.v_dino_i + g_opraw + g_D mid_i         (gradient reaching w_i)
//     g_opraw = [1e-6 <= sum w <= 1] (g_op - g_rgb.rgb_sky - g_F.dino_sky - g_depth sum(w mid) / op^2), g_D = g_depth/op
//   dL/dx_i = G_i T_i exp(-x_i) - sum_{k>i} (G_k w_k + g_T_k T_k)          (the reverse sweep of composite_bwd_kernel)
//   with r_s = sigma_s / (sigma + 1e-6):  d r_s_i = w_i (g_rgb.rgb_s_i (1 - sh_i) + g_F.dino_s_i)  (r_d likewise), and
//   d sigma_s += d r_s / (sigma + 1e-6),  d sigma -= (d r_s sigma_s + d r_d sigma_d) / (sigma + 1e-6)^2
#include "common.cuh"
#include "ray_scan.cuh"

namespace emer {

constexpr int RENDER_WARPS = 8;
constexpr int RENDER_MAX_PER_LANE = 8;     // feature channels C <= 256

__device__ __forceinline__ float ld(const float* p, int64_t i) { return __ldg(p + i); }

__global__ void __launch_bounds__(RENDER_WARPS * 32) render_fwd_kernel(const emer_render_in in,
                                                                       const emer_render_out out, bool decomp) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * RENDER_WARPS + (threadIdx.x >> 5);
    if (ray >= in.n_rays) return;
    const int S = in.n_samples, C = in.n_dino;
    const int64_t base = ray * S;
    const bool two = in.sigma_s != nullptr;
    const bool blend_rgb = !in.rgb && in.rgb_s;
    const bool blend_dino = !in.dino && in.dino_s;
    const bool has_dino = in.dino || in.dino_s;

    RayScan<true> scan;
    RayScan<false> scan_s, scan_d;
    float acc_rgb[3] = {0.0f, 0.0f, 0.0f}, acc_shr = 0.0f, acc_sh = 0.0f;
    float acc_srgb[3] = {0.0f, 0.0f, 0.0f}, acc_srs[3] = {0.0f, 0.0f, 0.0f}, acc_so[3] = {0.0f, 0.0f, 0.0f};
    float acc_drgb[3] = {0.0f, 0.0f, 0.0f}, acc_ff[3] = {0.0f, 0.0f, 0.0f}, acc_bf[3] = {0.0f, 0.0f, 0.0f};
    float acc_f[RENDER_MAX_PER_LANE], acc_fs[RENDER_MAX_PER_LANE], acc_fd[RENDER_MAX_PER_LANE];
#pragma unroll
    for (int j = 0; j < RENDER_MAX_PER_LANE; ++j) acc_f[j] = acc_fs[j] = acc_fd[j] = 0.0f;

    for (int s0 = 0; s0 < S; s0 += 32) {
        const int s = s0 + lane;
        const bool ok = s < S;
        const int64_t i = base + s;
        float a = 0.0f, b = 0.0f, sg = 0.0f;
        if (ok) {
            a = ld(in.t0, i);
            b = ld(in.t1, i);
            sg = ld(in.sigma, i);
        }
        float T;
        const float w = scan.step(a, b, sg, ok, s0, S, lane, T);
        if (ok) {
            if (out.weights) out.weights[i] = w;
            if (out.trans) out.trans[i] = T;
        }
        float rs = 0.0f, rd = 0.0f, ws = 0.0f, wd = 0.0f;
        if (two) {
            const float sgs = ok ? ld(in.sigma_s, i) : 0.0f;
            const float sgd = ok ? ld(in.sigma_d, i) : 0.0f;
            rs = sgs / (sg + 1e-6f);
            rd = sgd / (sg + 1e-6f);
            if (decomp) {
                float Ts, Td;
                ws = scan_s.step(a, b, sgs, ok, s0, S, lane, Ts);
                wd = scan_d.step(a, b, sgd, ok, s0, S, lane, Td);
            }
        }
        if (ok) {
            const float sh = in.shadow ? ld(in.shadow, i) : 0.0f;
            if (in.shadow) {
                acc_shr = fmaf(w, sh * sh, acc_shr);
                acc_sh = fmaf(w, sh, acc_sh);
            }
            if (in.rgb) {
#pragma unroll
                for (int k = 0; k < 3; ++k) acc_rgb[k] = fmaf(w, ld(in.rgb, i * 3 + k), acc_rgb[k]);
            } else if (blend_rgb) {
                const float om = 1.0f - sh;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const float cs = ld(in.rgb_s, i * 3 + k), cd = ld(in.rgb_d, i * 3 + k);
                    acc_rgb[k] = fmaf(w, rs * cs * om + rd * cd, acc_rgb[k]);
                    if (decomp) {
                        acc_srgb[k] = fmaf(ws, cs, acc_srgb[k]);
                        acc_srs[k] = fmaf(ws, cs * om, acc_srs[k]);
                        acc_so[k] = fmaf(ws, cs * sh, acc_so[k]);
                        acc_drgb[k] = fmaf(wd, cd, acc_drgb[k]);
                    }
                }
            }
            if (decomp && in.fwd_flow) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    acc_ff[k] = fmaf(wd, ld(in.fwd_flow, i * in.ld_flow + k), acc_ff[k]);
                    acc_bf[k] = fmaf(wd, ld(in.bwd_flow, i * in.ld_flow + k), acc_bf[k]);
                }
            }
        }
        if (has_dino) {
            const int n = min(32, S - s0);
            for (int k = 0; k < n; ++k) {
                const float wk = __shfl_sync(0xffffffffu, w, k);
                const float rsk = __shfl_sync(0xffffffffu, rs, k);
                const float rdk = __shfl_sync(0xffffffffu, rd, k);
                const float wsk = __shfl_sync(0xffffffffu, ws, k);
                const float wdk = __shfl_sync(0xffffffffu, wd, k);
                const int64_t row = (base + s0 + k) * C;
#pragma unroll
                for (int j = 0; j < RENDER_MAX_PER_LANE; ++j) {
                    const int c = lane + 32 * j;
                    if (c < C) {
                        if (blend_dino) {
                            const float ds = ld(in.dino_s, row + c), dd = ld(in.dino_d, row + c);
                            acc_f[j] = fmaf(wk, rsk * ds + rdk * dd, acc_f[j]);
                            if (decomp) {
                                acc_fs[j] = fmaf(wsk, ds, acc_fs[j]);
                                acc_fd[j] = fmaf(wdk, dd, acc_fd[j]);
                            }
                        } else {
                            acc_f[j] = fmaf(wk, ld(in.dino, row + c), acc_f[j]);
                        }
                    }
                }
            }
        }
    }

    // ---- ray totals (warp reductions on every lane; lane 0 writes the per-ray scalars)
    float op, dep, med;
    scan.finish(op, dep, med);
    float op_s = 0.0f, dep_s = 0.0f, op_d = 0.0f, dep_d = 0.0f, unused;
    if (decomp) {
        scan_s.finish(op_s, dep_s, unused);
        scan_d.finish(op_d, dep_d, unused);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        acc_rgb[k] = warp_sum(acc_rgb[k]);
        if (decomp) {
            acc_srgb[k] = warp_sum(acc_srgb[k]);
            acc_srs[k] = warp_sum(acc_srs[k]);
            acc_so[k] = warp_sum(acc_so[k]);
            acc_drgb[k] = warp_sum(acc_drgb[k]);
            acc_ff[k] = warp_sum(acc_ff[k]);
            acc_bf[k] = warp_sum(acc_bf[k]);
        }
    }
    acc_shr = warp_sum(acc_shr);
    acc_sh = warp_sum(acc_sh);
    if (lane == 0) {
        if (out.opacity) out.opacity[ray] = op;
        if (out.depth) out.depth[ray] = dep;
        if (out.median_depth) out.median_depth[ray] = med;
        if (out.shadow_ratio) out.shadow_ratio[ray] = acc_shr;
        if (out.static_opacity) out.static_opacity[ray] = op_s;
        if (out.static_depth) out.static_depth[ray] = dep_s;
        if (out.dynamic_opacity) out.dynamic_opacity[ray] = op_d;
        if (out.dynamic_depth) out.dynamic_depth[ray] = dep_d;
        if (out.shadow) out.shadow[ray] = acc_sh;
    }
    if (lane < 3) {
        // each of lanes 0..2 writes its colour channel (static indexing keeps the accumulators in registers)
        float v = lane == 0 ? acc_rgb[0] : lane == 1 ? acc_rgb[1] : acc_rgb[2];
        const float sky = in.rgb_sky ? ld(in.rgb_sky, ray * 3 + lane) : 0.0f;
        if (in.rgb_sky) v = v + sky * (1.0f - op);
        if (out.rgb) out.rgb[ray * 3 + lane] = v;
        auto pick = [lane](const float* x) { return lane == 0 ? x[0] : lane == 1 ? x[1] : x[2]; };
        if (out.static_rgb) {
            float sr = pick(acc_srgb);
            if (in.rgb_sky) sr = sr + sky * (1.0f - op_s);
            out.static_rgb[ray * 3 + lane] = sr;
        }
        if (out.dynamic_rgb) out.dynamic_rgb[ray * 3 + lane] = pick(acc_drgb);
        if (out.shadow_reduced_static_rgb) out.shadow_reduced_static_rgb[ray * 3 + lane] = pick(acc_srs);
        if (out.shadow_only_static_rgb) out.shadow_only_static_rgb[ray * 3 + lane] = pick(acc_so) + (1.0f - acc_sh);
        if (out.forward_flow) out.forward_flow[ray * 3 + lane] = pick(acc_ff);
        if (out.backward_flow) out.backward_flow[ray * 3 + lane] = pick(acc_bf);
    }
    if (has_dino) {
#pragma unroll
        for (int j = 0; j < RENDER_MAX_PER_LANE; ++j) {
            const int c = lane + 32 * j;
            if (c < C) {
                const int64_t o = ray * C + c;
                float f = acc_f[j];
                const float sky = in.dino_sky ? ld(in.dino_sky, o) : 0.0f;
                if (in.dino_sky) f = f + sky * (1.0f - op);
                if (out.dino_pe_free) out.dino_pe_free[o] = f;
                if (out.dino) out.dino[o] = in.dino_pe ? f + ld(in.dino_pe, o) : f;
                if (out.static_dino) out.static_dino[o] = in.dino_sky ? acc_fs[j] + sky * (1.0f - op) : acc_fs[j];
                if (out.dynamic_dino) out.dynamic_dino[o] = acc_fd[j];
            }
        }
    }
}

__global__ void __launch_bounds__(RENDER_WARPS * 32) render_bwd_kernel(const emer_render_in in,
                                                                       const float* __restrict__ weights,
                                                                       const float* __restrict__ trans,
                                                                       const emer_render_grad g) {
    const int lane = threadIdx.x & 31;
    const int64_t ray = (int64_t)blockIdx.x * RENDER_WARPS + (threadIdx.x >> 5);
    if (ray >= in.n_rays) return;
    const int S = in.n_samples, C = in.n_dino;
    const int64_t base = ray * S;
    const bool two = in.sigma_s != nullptr;
    const bool blend_rgb = !in.rgb && in.rgb_s;
    const bool blend_dino = !in.dino && in.dino_s;
    const bool has_dino = in.dino || in.dino_s;

    // ---- pass 1: ray totals, as composite_bwd_kernel
    float sum_w = 0.0f, sum_wm = 0.0f;
    for (int s = lane; s < S; s += 32) {
        const float w = ld(weights, base + s);
        const float mid = (ld(in.t0, base + s) + ld(in.t1, base + s)) / 2.0f;
        sum_w += w;
        sum_wm = fmaf(w, mid, sum_wm);
    }
    sum_w = warp_sum(sum_w);
    sum_wm = warp_sum(sum_wm);
    const float op = fminf(fmaxf(sum_w, 1e-6f), 1.0f);
    const float gd = g.g_depth ? ld(g.g_depth, ray) : 0.0f;
    const float go = g.g_opacity ? ld(g.g_opacity, ray) : 0.0f;
    float grgb[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) grgb[k] = g.g_rgb ? ld(g.g_rgb, ray * 3 + k) : 0.0f;
    const float gshr = g.g_shadow_ratio ? ld(g.g_shadow_ratio, ray) : 0.0f;

    // per-ray terms: the sky colour and features pull on the opacity; the PE gets g_dino as it is
    float g_sky = 0.0f;
    if (in.rgb_sky) {
#pragma unroll
        for (int k = 0; k < 3; ++k) g_sky = fmaf(grgb[k], ld(in.rgb_sky, ray * 3 + k), g_sky);
        if (g.d_rgb_sky && lane < 3) {
            const float gl = lane == 0 ? grgb[0] : lane == 1 ? grgb[1] : grgb[2];
            g.d_rgb_sky[ray * 3 + lane] = gl * (1.0f - op);
        }
    }
    float gF[RENDER_MAX_PER_LANE];
    float g_dsky = 0.0f;
#pragma unroll
    for (int j = 0; j < RENDER_MAX_PER_LANE; ++j) {
        const int c = lane + 32 * j;
        gF[j] = 0.0f;
        if (has_dino && c < C) {
            const int64_t o = ray * C + c;
            const float gdino = g.g_dino ? ld(g.g_dino, o) : 0.0f;
            gF[j] = g.g_dino_pe_free ? gdino + ld(g.g_dino_pe_free, o) : gdino;
            if (g.d_dino_pe) g.d_dino_pe[o] = gdino;
            if (in.dino_sky) {
                g_dsky = fmaf(gF[j], ld(in.dino_sky, o), g_dsky);
                if (g.d_dino_sky) g.d_dino_sky[o] = gF[j] * (1.0f - op);
            }
        }
    }
    if (has_dino && in.dino_sky) g_dsky = warp_sum(g_dsky);
    const float g_D = gd / op;                                   // depth = D / op
    const float g_op = go - g_sky - g_dsky - gd * sum_wm / (op * op);
    const float g_opraw = (sum_w >= 1e-6f && sum_w <= 1.0f) ? g_op : 0.0f;   // clamp passes in range

    // ---- pass 2: reverse sweep with a running suffix sum
    float carry = 0.0f;
    const int chunks = (S + 31) / 32;
    for (int ch = chunks - 1; ch >= 0; --ch) {
        const int s0 = ch * 32;
        const int s = s0 + lane;
        const bool ok = s < S;
        const int64_t i = base + s;
        float a = 0.0f, b = 0.0f, sg = 0.0f, w = 0.0f, T = 0.0f, gw = 0.0f, gT = 0.0f;
        float sgs = 0.0f, sgd = 0.0f, sh = 0.0f;
        if (ok) {
            a = ld(in.t0, i);
            b = ld(in.t1, i);
            sg = ld(in.sigma, i);
            w = ld(weights, i);
            T = ld(trans, i);
            if (g.g_weights) gw = ld(g.g_weights, i);
            if (g.g_trans) gT = ld(g.g_trans, i);
            if (two) {
                sgs = ld(in.sigma_s, i);
                sgd = ld(in.sigma_d, i);
            }
            if (in.shadow) sh = ld(in.shadow, i);
        }
        const float den = sg + 1e-6f;
        const float rs = two ? sgs / den : 0.0f;
        const float rd = two ? sgd / den : 0.0f;
        float gx = 0.0f;                   // g_rgb.v_rgb + g_shr sh^2 + g_F.v_dino: the gradient w_i gets from them
        float drs = 0.0f, drd = 0.0f;      // d loss / d r_s, d r_d
        if (ok) {
            float dsh = 0.0f;
            if (in.shadow) {
                gx = fmaf(gshr, sh * sh, gx);
                dsh = w * gshr * 2.0f * sh;
            }
            if (in.rgb) {
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    gx = fmaf(grgb[k], ld(in.rgb, i * 3 + k), gx);
                    if (g.d_rgb) g.d_rgb[i * 3 + k] = w * grgb[k];
                }
            } else if (blend_rgb) {
                const float om = 1.0f - sh;
                float cs_g = 0.0f, cd_g = 0.0f;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    cs_g = fmaf(grgb[k], ld(in.rgb_s, i * 3 + k), cs_g);
                    cd_g = fmaf(grgb[k], ld(in.rgb_d, i * 3 + k), cd_g);
                    if (g.d_rgb_s) g.d_rgb_s[i * 3 + k] = w * grgb[k] * rs * om;
                    if (g.d_rgb_d) g.d_rgb_d[i * 3 + k] = w * grgb[k] * rd;
                }
                gx = gx + (rs * cs_g * om + rd * cd_g);
                drs = w * cs_g * om;
                drd = w * cd_g;
                dsh = dsh - w * rs * cs_g;
            }
            if (g.d_shadow) g.d_shadow[i] = dsh;
        }
        if (has_dino) {
            float my_s = 0.0f, my_d = 0.0f;
            const int n = min(32, S - s0);
            for (int k = 0; k < n; ++k) {
                const float wk = __shfl_sync(0xffffffffu, w, k);
                const float rsk = __shfl_sync(0xffffffffu, rs, k);
                const float rdk = __shfl_sync(0xffffffffu, rd, k);
                const int64_t row = (base + s0 + k) * C;
                float ps = 0.0f, pd = 0.0f;
#pragma unroll
                for (int j = 0; j < RENDER_MAX_PER_LANE; ++j) {
                    const int c = lane + 32 * j;
                    if (c < C) {
                        const float wg = wk * gF[j];
                        if (blend_dino) {
                            ps = fmaf(gF[j], ld(in.dino_s, row + c), ps);
                            pd = fmaf(gF[j], ld(in.dino_d, row + c), pd);
                            if (g.d_dino_s) g.d_dino_s[row + c] = wg * rsk;
                            if (g.d_dino_d) g.d_dino_d[row + c] = wg * rdk;
                        } else {
                            ps = fmaf(gF[j], ld(in.dino, row + c), ps);
                            if (g.d_dino) g.d_dino[row + c] = wg;
                        }
                    }
                }
                ps = warp_sum(ps);
                if (blend_dino) pd = warp_sum(pd);
                if (lane == k) {
                    my_s = ps;
                    my_d = pd;
                }
            }
            if (blend_dino) {
                gx = gx + (rs * my_s + rd * my_d);
                drs = fmaf(w, my_s, drs);
                drd = fmaf(w, my_d, drd);
            } else {
                gx = gx + my_s;
            }
        }
        const float delta = b - a;
        const float mid = (a + b) / 2.0f;
        const float G = gw + gx + g_opraw + g_D * mid;
        const float q = ok ? fmaf(G, w, gT * T) : 0.0f;
        const float suf_incl = warp_scan_incl_rev(q, lane);
        const float suffix_excl = carry + warp_scan_excl_rev(suf_incl, lane);
        const float ex = expf(-(sg * delta));
        const float dx = G * T * ex - suffix_excl;
        if (ok) {
            float dsig = dx * delta;
            if (two) {
                dsig = dsig - (drs * sgs + drd * sgd) / (den * den);
                if (g.d_sigma_s) g.d_sigma_s[i] = drs / den;
                if (g.d_sigma_d) g.d_sigma_d[i] = drd / den;
            }
            if (g.d_sigma) g.d_sigma[i] = dsig;
        }
        carry += __shfl_sync(0xffffffffu, suf_incl, 0);
    }
}

static int check_render_in(const emer_render_in* in, const char* what) {
    EMER_REQUIRE(in && in->t0 && in->t1 && in->sigma, "%s: NULL pointer", what);
    EMER_REQUIRE(in->n_samples >= 1, "%s: n_samples must be >= 1", what);
    EMER_REQUIRE(!in->sigma_s == !in->sigma_d, "%s: sigma_s and sigma_d come together", what);
    EMER_REQUIRE(!in->rgb_s == !in->rgb_d && (!in->rgb_s || in->sigma_s),
                 "%s: rgb_s and rgb_d come together, with sigma_s and sigma_d", what);
    EMER_REQUIRE(!in->dino_s == !in->dino_d && (!in->dino_s || in->sigma_s),
                 "%s: dino_s and dino_d come together, with sigma_s and sigma_d", what);
    EMER_REQUIRE(!(in->dino || in->dino_s) || (in->n_dino >= 1 && in->n_dino <= 32 * RENDER_MAX_PER_LANE),
                 "%s: feature channels %d out of range", what, in->n_dino);
    EMER_REQUIRE(!in->fwd_flow == !in->bwd_flow && (!in->fwd_flow || in->ld_flow >= 3),
                 "%s: flows need both directions and a row stride >= 3", what);
    return 0;
}

}  // namespace emer

using namespace emer;

extern "C" int emer_render_fwd(const emer_render_in* in, const emer_render_out* out, void* stream) {
    EMER_REQUIRE(in && out, "emer_render_fwd: NULL pointer");
    if (in->n_rays == 0) return 0;
    if (int rc = check_render_in(in, "emer_render_fwd")) return rc;
    const bool decomp = out->static_opacity || out->dynamic_opacity || out->static_depth || out->dynamic_depth ||
                        out->static_rgb || out->dynamic_rgb || out->shadow_reduced_static_rgb ||
                        out->shadow_only_static_rgb || out->shadow || out->forward_flow || out->backward_flow ||
                        out->static_dino || out->dynamic_dino;
    EMER_REQUIRE(!decomp || in->sigma_s, "emer_render_fwd: the decomposition needs sigma_s and sigma_d");
    EMER_REQUIRE(!(out->static_rgb || out->dynamic_rgb || out->shadow_reduced_static_rgb ||
                   out->shadow_only_static_rgb) || (in->rgb_s && !in->rgb),
                 "emer_render_fwd: static / dynamic colours need rgb_s and rgb_d (and no rgb)");
    EMER_REQUIRE(!(out->shadow_reduced_static_rgb || out->shadow_only_static_rgb || out->shadow || out->shadow_ratio) ||
                     in->shadow, "emer_render_fwd: shadow outputs need the shadow input");
    EMER_REQUIRE(!(out->forward_flow || out->backward_flow) || in->fwd_flow, "emer_render_fwd: flow outputs need flows");
    EMER_REQUIRE(!(out->static_dino || out->dynamic_dino) || (in->dino_s && !in->dino),
                 "emer_render_fwd: static / dynamic features need dino_s and dino_d (and no dino)");
    EMER_REQUIRE(!(out->rgb) || in->rgb || in->rgb_s, "emer_render_fwd: rgb needs a colour input");
    EMER_REQUIRE(!(out->dino || out->dino_pe_free) || in->dino || in->dino_s, "emer_render_fwd: dino needs features");
    render_fwd_kernel<<<(unsigned)ceil_div(in->n_rays, RENDER_WARPS), RENDER_WARPS * 32, 0, (cudaStream_t)stream>>>(
        *in, *out, decomp);
    return check_launch("emer_render_fwd");
}

extern "C" int emer_render_bwd(const emer_render_in* in, const float* weights, const float* trans,
                               const emer_render_grad* grad, void* stream) {
    EMER_REQUIRE(in && grad, "emer_render_bwd: NULL pointer");
    if (in->n_rays == 0) return 0;
    if (int rc = check_render_in(in, "emer_render_bwd")) return rc;
    EMER_REQUIRE(weights && trans, "emer_render_bwd: NULL weights or trans");
    render_bwd_kernel<<<(unsigned)ceil_div(in->n_rays, RENDER_WARPS), RENDER_WARPS * 32, 0, (cudaStream_t)stream>>>(
        *in, weights, trans, *grad);
    return check_launch("emer_render_bwd");
}
