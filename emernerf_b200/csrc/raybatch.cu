// A training batch of pixel rays drawn on the device: ScenePixelSource.get_train_rays
// (datasets/base/pixel_source.py:564-731) without a host sync.
//
// emer_topk_ratio is the selection half of torch.multinomial(p[cand].reshape(-1), k, replacement=False), which ATen
// computes as topk(p / q, k) with q ~ Exp(1) drawn by the caller: the k largest keys p[cand[j / plane], j % plane] / q[j]
// (IEEE division), ordered by descending key, then ascending j.  The keys are finite and non-negative (the caller
// validates p as torch does; q > 0), so their fp32 bit patterns, with the sign of -0 cleared, order like the keys.
//   1-3. topk_hist_kernel, passes 0-2: a radix select on the bit pattern, digits of 11, 11 and 10 bits.  Every CTA counts the
//        digits of the keys in its contiguous chunk of j that match the threshold's bits known so far, adds its
//        histogram into the workspace (integer atomics), and the CTA that takes the last ticket (cta_reduce.cuh) picks
//        the digit that holds the k-th largest key and zeroes the histogram.  After pass 3 the k-th largest key T and
//        the number r of keys equal to T that belong to the top k are known.
//   4.   topk_collect_kernel: every key > T (fewer than k) is appended to the survivor list; each CTA counts its keys
//        equal to T.
//   5.   topk_sort_kernel, one CTA: loads the survivors, appends the r keys equal to T of smallest j (walking the CTAs'
//        chunks in order and rescanning only chunks that hold needed ties), bitonic-sorts the k (key, ~j) pairs in
//        shared memory and writes j.
// Launches 1-4 each read p (through cand) and q once: 11.5 MB at 1.44 M keys, L2-resident after the first.
// Bounds: 1 <= k <= EMER_TOPK_MAX_K (16 384 pairs of 8 bytes = 128 KB of shared memory), k <= M < 2^31.
//
// emer_pixel_batch turns the uniform draws and the selected indices into the batch in one launch: the importance rays'
// idx_to_3d (:19-36), upscaling, offset and clamp (:594-613), the gathers of :699-716 and the ray of pixel_ray
// (rays.cuh, shared with emer_gen_rays).
#include "cta_reduce.cuh"
#include "rays.cuh"

namespace emer {

constexpr int SEL_THREADS = 512;
constexpr int SEL_MAX_CTAS = 512;
constexpr int SORT_THREADS = 1024;
constexpr int RADIX_BINS = 2048;

// workspace layout, in 32-bit words (EMER_RAYBATCH_WORKSPACE_BYTES)
constexpr int WS_HIST = 0;                         // [RADIX_BINS] digit counts of the current pass
constexpr int WS_TICKET = RADIX_BINS;              // cta_reduce.cuh ticket
constexpr int WS_PREFIX = RADIX_BINS + 1;          // bits of T known so far
constexpr int WS_KREM = RADIX_BINS + 2;            // rank of T among the keys that match those bits
constexpr int WS_NGT = RADIX_BINS + 3;             // survivors appended by topk_collect_kernel
constexpr int WS_EQ = RADIX_BINS + 16;             // [SEL_MAX_CTAS] keys equal to T per CTA
constexpr int WS_SURV = WS_EQ + SEL_MAX_CTAS;      // [EMER_TOPK_MAX_K] uint64 survivors (8-byte aligned)
static_assert(WS_SURV % 2 == 0, "survivors must be 8-byte aligned");
static_assert((WS_SURV + 2 * EMER_TOPK_MAX_K) * 4 == EMER_RAYBATCH_WORKSPACE_BYTES, "workspace size");

__device__ __forceinline__ uint32_t ratio_key(const float* __restrict__ p, uint32_t plane,
                                              const int64_t* __restrict__ cand, const float* __restrict__ q,
                                              uint32_t j) {
    const uint32_t c = j / plane;
    const float v = __ldg(p + __ldg(cand + c) * (int64_t)plane + (j - c * plane));
    return __float_as_uint(__fdiv_rn(v, __ldg(q + j))) & 0x7fffffffu;
}

// (key, j) as one integer that orders like (key descending, j ascending) when sorted descending
__device__ __forceinline__ uint64_t pair_of(uint32_t key, uint32_t j) { return ((uint64_t)key << 32) | (uint32_t)~j; }

// pass 0, 1, 2: the digit of bits [shift, shift + bits) = [21, 32), [10, 21), [0, 10)
__global__ void __launch_bounds__(SEL_THREADS) topk_hist_kernel(const float* __restrict__ p, uint32_t plane,
                                                               const int64_t* __restrict__ cand,
                                                               const float* __restrict__ q, uint32_t m,
                                                               uint32_t chunk, uint32_t k, int pass, uint32_t* ws) {
    const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
    const int nb = pass == 2 ? 1024 : 2048;
    const int high = pass == 0 ? 31 : shift + (pass == 2 ? 10 : 11);    // bits at and above high are known
    constexpr int PER = RADIX_BINS / SEL_THREADS;
    __shared__ uint32_t h[RADIX_BINS];
    __shared__ uint32_t warp_tot[SEL_THREADS / 32];
    for (int b = threadIdx.x; b < nb; b += SEL_THREADS) h[b] = 0u;
    const uint32_t prefix = pass == 0 ? 0u : __ldcg(ws + WS_PREFIX);
    __syncthreads();
    const uint32_t begin = blockIdx.x * chunk, end = min(m, begin + chunk);
    for (uint32_t j = begin + threadIdx.x; j < end; j += SEL_THREADS) {
        const uint32_t key = ratio_key(p, plane, cand, q, j);
        if ((key >> high) == (prefix >> high)) atomicAdd(&h[(key >> shift) & (nb - 1)], 1u);
    }
    __syncthreads();
    for (int b = threadIdx.x; b < nb; b += SEL_THREADS)
        if (h[b]) atomicAdd(ws + WS_HIST + b, h[b]);
    if (!take_last_ticket(ws + WS_TICKET)) return;

    // The last CTA: thread t holds bins [t*PER, t*PER + PER); the counts above its bins are the sum over threads > t.
    const uint32_t krem = pass == 0 ? k : __ldcg(ws + WS_KREM);
    uint32_t c[PER], s = 0u;
#pragma unroll
    for (int e = 0; e < PER; ++e) {
        const int b = threadIdx.x * PER + e;
        c[e] = b < nb ? __ldcg(ws + WS_HIST + b) : 0u;
        if (b < nb) ws[WS_HIST + b] = 0u;
        s += c[e];
    }
    // inclusive scan in descending thread order
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    uint32_t incl = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t v = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += v;
    }
    if (lane == 0) warp_tot[wid] = incl;
    __syncthreads();
    uint32_t above = incl - s;
    for (int w = wid + 1; w < SEL_THREADS / 32; ++w) above += warp_tot[w];
    if (above < krem && krem <= above + s) {
#pragma unroll
        for (int e = PER - 1; e >= 0; --e) {
            if (krem <= above + c[e]) {
                ws[WS_PREFIX] = prefix | ((uint32_t)(threadIdx.x * PER + e) << shift);
                ws[WS_KREM] = krem - above;
                break;
            }
            above += c[e];
        }
    }
    release_ticket(ws + WS_TICKET);
}

__global__ void __launch_bounds__(SEL_THREADS) topk_collect_kernel(const float* __restrict__ p, uint32_t plane,
                                                                  const int64_t* __restrict__ cand,
                                                                  const float* __restrict__ q, uint32_t m,
                                                                  uint32_t chunk, uint32_t* ws) {
    __shared__ uint32_t sh[SEL_THREADS / 32];
    const uint32_t t = __ldcg(ws + WS_PREFIX);
    uint64_t* surv = reinterpret_cast<uint64_t*>(ws + WS_SURV);
    const uint32_t begin = blockIdx.x * chunk, end = min(m, begin + chunk);
    uint32_t eq = 0u;
    for (uint32_t j = begin + threadIdx.x; j < end; j += SEL_THREADS) {
        const uint32_t key = ratio_key(p, plane, cand, q, j);
        if (key > t) surv[atomicAdd(ws + WS_NGT, 1u)] = pair_of(key, j);
        eq += key == t;
    }
    eq = block_sum<SEL_THREADS / 32>(eq, sh);
    if (threadIdx.x == 0) ws[WS_EQ + blockIdx.x] = eq;
}

__global__ void __launch_bounds__(SORT_THREADS) topk_sort_kernel(const float* __restrict__ p, uint32_t plane,
                                                                const int64_t* __restrict__ cand,
                                                                const float* __restrict__ q, uint32_t m,
                                                                uint32_t chunk, uint32_t n_ctas, uint32_t k,
                                                                uint32_t n_sort, uint32_t* ws,
                                                                int64_t* __restrict__ out_idx) {
    extern __shared__ uint64_t pairs[];
    __shared__ uint32_t warp_cnt[SORT_THREADS / 32];
    __shared__ uint32_t eq_cta;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t t = __ldcg(ws + WS_PREFIX);
    const uint32_t n_gt = __ldcg(ws + WS_NGT);
    uint64_t* surv = reinterpret_cast<uint64_t*>(ws + WS_SURV);
    for (uint32_t i = threadIdx.x; i < n_gt; i += SORT_THREADS) {
        pairs[i] = __ldcg(surv + i);
        surv[i] = 0ull;
    }
    for (uint32_t i = k + threadIdx.x; i < n_sort; i += SORT_THREADS) pairs[i] = 0ull;   // below every real pair

    // the k - n_gt keys equal to T with the smallest j, in order of j
    uint32_t filled = n_gt;
    for (uint32_t b = 0; b < n_ctas && filled < k; ++b) {
        if (threadIdx.x == 0) eq_cta = __ldcg(ws + WS_EQ + b);
        __syncthreads();
        const uint32_t eq = eq_cta;
        __syncthreads();
        if (eq == 0u) continue;
        const uint32_t begin = b * chunk, end = min(m, begin + chunk);
        for (uint32_t base = begin; base < end && filled < k; base += SORT_THREADS) {
            const uint32_t j = base + threadIdx.x;
            const bool hit = j < end && ratio_key(p, plane, cand, q, j) == t;
            const unsigned ballot = __ballot_sync(0xffffffffu, hit);
            if (lane == 0) warp_cnt[wid] = __popc(ballot);
            __syncthreads();
            uint32_t rank = __popc(ballot & ((1u << lane) - 1u)), total = 0u;
            for (int w = 0; w < SORT_THREADS / 32; ++w) {
                rank += w < wid ? warp_cnt[w] : 0u;
                total += warp_cnt[w];
            }
            if (hit && filled + rank < k) pairs[filled + rank] = pair_of(t, j);
            filled = min(k, filled + total);
            __syncthreads();
        }
    }
    for (uint32_t b = threadIdx.x; b < n_ctas; b += SORT_THREADS) ws[WS_EQ + b] = 0u;
    if (threadIdx.x == 0) {
        ws[WS_NGT] = 0u;
        ws[WS_PREFIX] = 0u;
        ws[WS_KREM] = 0u;
    }
    __syncthreads();

    // bitonic sort, descending
    for (uint32_t size = 2; size <= n_sort; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t e = threadIdx.x; e < n_sort / 2; e += SORT_THREADS) {
                const uint32_t i = 2 * e - (e & (stride - 1)), o = i + stride;
                const uint64_t a = pairs[i], c = pairs[o];
                if (((i & size) == 0) ? (a < c) : (a > c)) {
                    pairs[i] = c;
                    pairs[o] = a;
                }
            }
            __syncthreads();
        }
    }
    for (uint32_t i = threadIdx.x; i < k; i += SORT_THREADS) out_idx[i] = (int64_t)(uint32_t)~(uint32_t)pairs[i];
}

constexpr int BATCH_THREADS = 128;

__global__ void __launch_bounds__(BATCH_THREADS) pixel_batch_kernel(const EmerPixelBatchIn a, const EmerPixelBatchOut o) {
    __shared__ int64_t feat_row[BATCH_THREADS];
    const int64_t n = a.n_uniform + a.n_importance;
    const int64_t i0 = (int64_t)blockIdx.x * BATCH_THREADS, i = i0 + threadIdx.x;
    if (i < n) {
        int64_t img, y, x;
        if (i < a.n_uniform) {
            img = __ldg(a.cand + __ldg(a.u_pick + i));
            y = __ldg(a.u_y + i);
            x = __ldg(a.u_x + i);
        } else {
            // idx_to_3d, then (row, col) * ds + offset, clamped to the image (pixel_source.py:594-613)
            const int64_t t = i - a.n_uniform, j = __ldg(a.i_sel + t);
            const int64_t plane = (int64_t)a.map_h * a.map_w;
            const int64_t c = j / plane, rem = j - c * plane, row = rem / a.map_w, col = rem - row * a.map_w;
            img = __ldg(a.cand + c);
            y = min(max(row * a.map_downscale + __ldg(a.i_dy + t), (int64_t)0), (int64_t)a.height - 1);
            x = min(max(col * a.map_downscale + __ldg(a.i_dx + t), (int64_t)0), (int64_t)a.width - 1);
        }
        const int64_t pix = (img * a.height + y) * a.width + x;
        o.img_idx[i] = img;
        if (o.cam_idx) o.cam_idx[i] = __ldg(a.cam_ids + img);
        if (o.pixels) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) o.pixels[i * 3 + ch] = __ldg(a.images + pix * 3 + ch);
        }
        if (o.sky_masks) o.sky_masks[i] = __ldg(a.sky_masks + pix);
        if (o.dynamic_masks) o.dynamic_masks[i] = __ldg(a.dynamic_masks + pix);
        if (o.timestamps) o.timestamps[i] = __ldg(a.timestamps + img);
        const float fx = (float)x, fy = (float)y;
        float org[3], dir[3], nrm;
        pixel_ray(a.c2w + img * 16, a.intrinsics + img * 9, fx, fy, org, dir, nrm);
#pragma unroll
        for (int r = 0; r < 3; ++r) {
            o.origins[i * 3 + r] = org[r];
            o.viewdirs[i * 3 + r] = dir[r];
        }
        o.norms[i] = nrm;
        o.pixel_coords[i * 2 + 0] = pixel_coord(fy, a.height);
        o.pixel_coords[i * 2 + 1] = pixel_coord(fx, a.width);
        if (o.features) {
            const int64_t fr = feature_cell(fy, a.feat_scale_y, a.feat_h);
            const int64_t fc = feature_cell(fx, a.feat_scale_x, a.feat_w);
            feat_row[threadIdx.x] = ((img * a.feat_h + fr) * a.feat_w + fc) * a.feat_c;
        }
    }
    if (!o.features) return;
    __syncthreads();
    copy_feature_rows(a.features, feat_row, (int)min((int64_t)BATCH_THREADS, n - i0), a.feat_c,
                      o.features + i0 * a.feat_c, BATCH_THREADS);
}

}  // namespace emer

using namespace emer;

extern "C" int emer_topk_ratio(const float* p, int64_t plane, const int64_t* cand, int64_t n_cand, const float* q,
                               int64_t k, int64_t* out_idx, void* workspace, void* stream) {
    EMER_REQUIRE(p && cand && q && out_idx && workspace, "emer_topk_ratio: NULL pointer");
    EMER_REQUIRE(plane > 0 && n_cand > 0, "emer_topk_ratio: empty map");
    const int64_t m = plane * n_cand;
    EMER_REQUIRE(m < ((int64_t)1 << 31), "emer_topk_ratio: %lld keys, the limit is 2^31 - 1", (long long)m);
    EMER_REQUIRE(k >= 1 && k <= EMER_TOPK_MAX_K && k <= m, "emer_topk_ratio: k = %lld outside [1, min(%d, %lld)]",
                 (long long)k, EMER_TOPK_MAX_K, (long long)m);
    cudaStream_t s = (cudaStream_t)stream;
    uint32_t* ws = (uint32_t*)workspace;
    const int64_t want_ctas = ceil_div(m, SEL_THREADS * 8);
    const uint32_t n_ctas = (uint32_t)(want_ctas < SEL_MAX_CTAS ? want_ctas : SEL_MAX_CTAS);
    const uint32_t chunk = (uint32_t)ceil_div(m, n_ctas);
    const uint32_t um = (uint32_t)m, upl = (uint32_t)plane, uk = (uint32_t)k;
    for (int pass = 0; pass < 3; ++pass)
        topk_hist_kernel<<<n_ctas, SEL_THREADS, 0, s>>>(p, upl, cand, q, um, chunk, uk, pass, ws);
    topk_collect_kernel<<<n_ctas, SEL_THREADS, 0, s>>>(p, upl, cand, q, um, chunk, ws);
    uint32_t n_sort = 2;
    while (n_sort < uk) n_sort <<= 1;
    const size_t smem = (size_t)n_sort * sizeof(uint64_t);
    static bool smem_set[64] = {};
    bool& set = smem_set[current_device()];
    if (!set) {
        cudaError_t e = cudaFuncSetAttribute(topk_sort_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                             EMER_TOPK_MAX_K * (int)sizeof(uint64_t));
        EMER_REQUIRE(e == cudaSuccess, "emer_topk_ratio: %s", cudaGetErrorString(e));
        set = true;
    }
    topk_sort_kernel<<<1, SORT_THREADS, smem, s>>>(p, upl, cand, q, um, chunk, n_ctas, uk, n_sort, ws, out_idx);
    return check_launch("emer_topk_ratio");
}

extern "C" int emer_pixel_batch(const EmerPixelBatchIn* in, const EmerPixelBatchOut* out, void* stream) {
    EMER_REQUIRE(in && out, "emer_pixel_batch: NULL argument");
    const int64_t n = in->n_uniform + in->n_importance;
    if (n == 0) return 0;
    EMER_REQUIRE(in->n_uniform >= 0 && in->n_importance >= 0, "emer_pixel_batch: negative ray count");
    EMER_REQUIRE(in->cand && in->c2w && in->intrinsics && out->img_idx && out->origins && out->viewdirs && out->norms &&
                     out->pixel_coords, "emer_pixel_batch: NULL pointer");
    EMER_REQUIRE(in->height > 0 && in->width > 0, "emer_pixel_batch: empty image");
    EMER_REQUIRE(in->n_uniform == 0 || (in->u_pick && in->u_x && in->u_y), "emer_pixel_batch: NULL uniform draws");
    EMER_REQUIRE(in->n_importance == 0 || (in->i_sel && in->i_dy && in->i_dx && in->map_h > 0 && in->map_w > 0),
                 "emer_pixel_batch: NULL importance draws");
    EMER_REQUIRE(!out->pixels || in->images, "emer_pixel_batch: pixels without images");
    EMER_REQUIRE(!out->sky_masks || in->sky_masks, "emer_pixel_batch: sky masks without a source");
    EMER_REQUIRE(!out->dynamic_masks || in->dynamic_masks, "emer_pixel_batch: dynamic masks without a source");
    EMER_REQUIRE(!out->timestamps || in->timestamps, "emer_pixel_batch: timestamps without a source");
    EMER_REQUIRE(!out->cam_idx || in->cam_ids, "emer_pixel_batch: camera ids without a source");
    EMER_REQUIRE(!out->features || (in->features && in->feat_h > 0 && in->feat_w > 0 && in->feat_c > 0 &&
                                    in->feat_c <= EMER_PIXEL_BATCH_MAX_FEATURES),
                 "emer_pixel_batch: features need a [N, h, w, C] map with 1 <= C <= %d", EMER_PIXEL_BATCH_MAX_FEATURES);
    pixel_batch_kernel<<<(unsigned)ceil_div(n, BATCH_THREADS), BATCH_THREADS, 0, (cudaStream_t)stream>>>(*in, *out);
    return check_launch("emer_pixel_batch");
}
