// The training losses of the reference's loss/base.py, value and gradient, one launch each way per loss call.
//
// Reference: RealValueLoss (:83-146), SkyLoss (:149-185), DepthLoss (:188-269), LineOfSightLoss (:272-335) with
// compute_line_of_sight_loss (:430-464), DynamicRegularizationLoss (:338-410), and the flow variants' cycle loss with
// its four flow statistics (train_emernerf.py:700-740).  Op by op those are elementwise torch
// calls, masks, boolean indexing (DepthLoss: a nonzero and a device-to-host sync) and means; the line-of-sight loss
// alone is ~30 launches each way.  Here:
//   forward : grid-stride pass over the elements (pointwise) or one warp per ray (per-ray sums over the S samples);
//             per-CTA partial sums go to the workspace, and the CTA that takes the last ticket sums them in CTA order,
//             writes out[0] = loss value and out[1] = the count the mean divides by, and resets the ticket.  No float
//             atomics: the same inputs on the same device give bit-identical values.
//   backward: one elementwise pass; the upstream gradient g is read from device memory and the count from out[1].
// Arithmetic is fp32 in the reference's op order; the Python-float constants arrive rounded once from double by the
// caller (as torch rounds Python scalars).
#include "common.cuh"
#include "cta_reduce.cuh"

namespace emer {

constexpr int LOSS_THREADS = 256;
constexpr int LOSS_WARPS = LOSS_THREADS / 32;
constexpr int LOSS_MAX_CTAS = 512;

struct LossWorkspace {
    unsigned int ticket;             // zero between calls: the last CTA resets it
    unsigned int pad[15];
    float sum_a[LOSS_MAX_CTAS];
    union {
        struct {
            float sum_b[LOSS_MAX_CTAS];
            long long count[LOSS_MAX_CTAS];
        };
        unsigned int norm_max[4][LOSS_MAX_CTAS];     // the cycle loss's four statistics (it needs no sum_b / count)
    };
};
static_assert(sizeof(LossWorkspace) <= EMER_LOSS_WORKSPACE_BYTES, "workspace layout exceeds the ABI size");

struct LossParams {
    int kind;
    const float* a;          // pointwise: prediction / opacity / density;  per ray: weights [R, S]
    const float* b;          // pointwise: target / sky mask / static density (or null);  per ray: t_vals [R, S] (or null)
    const float* c;          // per ray: gt depth / sky mask [R]
    int64_t n;               // pointwise: elements;  per ray: rays
    int s;                   // per ray: samples
    float p0, p1, p2;        // kind constants (see the entry points)
    float pre, post;         // per-element factor before the mean, factor after it
    float* out;              // [2]: value, count
    LossWorkspace* ws;
    const float* g;          // backward: upstream gradient (device scalar)
    float* da;
    float* db;
    const float* live;       // per-ray kinds, live entry points: one {p0, p1, p2, pre} for the launch, else null
};

// the per-step constants of a live call replace the launch's; a float call keeps its own
__device__ __forceinline__ LossParams with_live(LossParams p) {
    if (p.live) {
        p.p0 = __ldg(p.live);
        p.p1 = __ldg(p.live + 1);
        p.p2 = __ldg(p.live + 2);
        p.pre = __ldg(p.live + 3);
    }
    return p;
}

// ---------------------------------------------------------------------------------------------- the terms
__device__ __forceinline__ float real_term(int base, float d) {       // base: 0 l1, 1 l2, 2 smooth_l1 (beta 1)
    if (base == 0) return fabsf(d);
    if (base == 1) return d * d;
    const float z = fabsf(d);
    return z < 1.0f ? 0.5f * z * z / 1.0f : z - 0.5f * 1.0f;
}

__device__ __forceinline__ float real_grad(int base, float d, float gs) {
    if (base == 0) return d > 0.0f ? gs : (d < 0.0f ? -gs : 0.0f);
    if (base == 1) return 2.0f * d * gs;
    if (d <= -1.0f) return -gs;
    if (d >= 1.0f) return gs;
    return d * gs / 1.0f;
}

__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }

__device__ __forceinline__ bool depth_valid(float gt, float max_depth) { return gt > 0.01f && gt < max_depth; }

// -(c log c) + -(1 - c) log(1 - c), c = clamp(ratio^k, 1e-6, 1 - 1e-6), ratio = dyn / (dyn + st + 1e-7)
__device__ __forceinline__ float skewed_ratio(float r, float k) { return k == 2.0f ? r * r : powf(r, k); }

__device__ __forceinline__ float entropy_term(float dyn, float st, float k) {
    const float r = dyn / (dyn + st + 1e-7f);
    const float c = fminf(fmaxf(skewed_ratio(r, k), 1e-6f), 1.0f - 1e-6f);
    return -(c * logf(c)) + -(1.0f - c) * logf(1.0f - c);
}

// element i of a pointwise loss: (term, counted)
__device__ __forceinline__ float pointwise_term(const LossParams& p, int64_t i, bool& counted) {
    counted = true;
    const float a = __ldg(p.a + i);
    switch (p.kind) {
        case EMER_LOSS_L1: case EMER_LOSS_L2: case EMER_LOSS_SMOOTH_L1:
            return real_term(p.kind - EMER_LOSS_L1, a - __ldg(p.b + i)) * p.pre;
        case EMER_LOSS_DEPTH_L1: case EMER_LOSS_DEPTH_L2: case EMER_LOSS_DEPTH_SMOOTH_L1: {
            const float gt = __ldg(p.b + i);
            counted = depth_valid(gt, p.p0);
            if (!counted) return 0.0f;
            return real_term(p.kind - EMER_LOSS_DEPTH_L1, clamp01(a / p.p0) - clamp01(gt / p.p0));
        }
        case EMER_LOSS_SKY_BCE: {
            const float t = 1.0f - __ldg(p.b + i);
            return (t - 1.0f) * fmaxf(logf(1.0f - a), -100.0f) - t * fmaxf(logf(a), -100.0f);
        }
        case EMER_LOSS_SPARSITY:
            return a;
        default:   // EMER_LOSS_ENTROPY
            return entropy_term(a, __ldg(p.b + i), p.p0);
    }
}

// ---------------------------------------------------------------------------------------------- reduction
// Every CTA publishes its partials; the one that takes the last ticket adds them up in CTA order.  Returns true in
// thread 0 of that CTA, with the totals in a / b / c.
__device__ bool reduce_across_ctas(LossWorkspace* ws, float& a, float& b, long long& c) {
    __shared__ float shf[LOSS_WARPS];
    __shared__ long long shc[LOSS_WARPS];
    a = block_sum<LOSS_WARPS>(a, shf);
    b = block_sum<LOSS_WARPS>(b, shf);
    c = block_sum<LOSS_WARPS>(c, shc);
    if (threadIdx.x == 0) {
        ws->sum_a[blockIdx.x] = a;
        ws->sum_b[blockIdx.x] = b;
        ws->count[blockIdx.x] = c;
    }
    if (!take_last_ticket(&ws->ticket)) return false;
    a = 0.0f; b = 0.0f; c = 0;
    for (int i = threadIdx.x; i < (int)gridDim.x; i += LOSS_THREADS) {
        a += __ldcg(ws->sum_a + i);
        b += __ldcg(ws->sum_b + i);
        c += __ldcg(ws->count + i);
    }
    a = block_sum<LOSS_WARPS>(a, shf);
    b = block_sum<LOSS_WARPS>(b, shf);
    c = block_sum<LOSS_WARPS>(c, shc);
    release_ticket(&ws->ticket);
    return threadIdx.x == 0;
}

__global__ void __launch_bounds__(LOSS_THREADS) pointwise_loss_fwd_kernel(const LossParams p) {
    float sum = 0.0f;
    long long cnt = 0;
    for (int64_t i = (int64_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * LOSS_THREADS) {
        bool counted;
        const float v = pointwise_term(p, i, counted);
        if (counted) { sum += v; ++cnt; }
    }
    float unused = 0.0f;
    if (reduce_across_ctas(p.ws, sum, unused, cnt)) {
        const float count = (float)cnt;
        p.out[0] = sum / count * p.post;          // mean (NaN over no element, as torch's), then the coefficient
        p.out[1] = count;
    }
}

__global__ void __launch_bounds__(LOSS_THREADS) pointwise_loss_bwd_kernel(const LossParams p) {
    const float gs = __ldg(p.g) * p.post / __ldg(p.out + 1) * p.pre;      // d loss / d term, as autograd chains it
    for (int64_t i = (int64_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * LOSS_THREADS) {
        const float a = __ldg(p.a + i);
        switch (p.kind) {
            case EMER_LOSS_L1: case EMER_LOSS_L2: case EMER_LOSS_SMOOTH_L1:
                p.da[i] = real_grad(p.kind - EMER_LOSS_L1, a - __ldg(p.b + i), gs);
                break;
            case EMER_LOSS_DEPTH_L1: case EMER_LOSS_DEPTH_L2: case EMER_LOSS_DEPTH_SMOOTH_L1: {
                const float gt = __ldg(p.b + i);
                float d = 0.0f;
                if (depth_valid(gt, p.p0)) {
                    const float x = a / p.p0;
                    const float dl = real_grad(p.kind - EMER_LOSS_DEPTH_L1, clamp01(x) - clamp01(gt / p.p0), gs);
                    d = (x >= 0.0f && x <= 1.0f) ? dl / p.p0 : 0.0f;          // clamp passes on the closed interval
                }
                p.da[i] = d;
                break;
            }
            case EMER_LOSS_SKY_BCE: {
                const float t = 1.0f - __ldg(p.b + i);
                p.da[i] = gs * (a - t) / fmaxf((1.0f - a) * a, 1e-12f);
                break;
            }
            case EMER_LOSS_SPARSITY:
                p.da[i] = gs;
                break;
            default: {   // EMER_LOSS_ENTROPY: through clamp, pow, the ratio and its denominator
                const float st = __ldg(p.b + i);
                const float den = a + st + 1e-7f;
                const float r = a / den;
                const float sk = skewed_ratio(r, p.p0);
                const float c = fminf(fmaxf(sk, 1e-6f), 1.0f - 1e-6f);
                // summed in the order autograd accumulates the four uses of c: near c = 1 the log(1 - c) terms
                // dominate and the order shows in the last bits
                const float dc = gs * logf(1.0f - c) - gs * -(1.0f - c) / (1.0f - c) + -gs * logf(c) + -gs * c / c;
                const float dsk = (sk >= 1e-6f && sk <= 1.0f - 1e-6f) ? dc : 0.0f;
                const float dr = dsk * (p.p0 == 2.0f ? 2.0f * r : p.p0 * powf(r, p.p1));
                const float dden = -dr * (r / den);                          // torch's div backward
                if (p.da) p.da[i] = dr / den + dden;
                if (p.db) p.db[i] = dden;
                break;
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- per-ray sums
// line of sight (p0 = epsilon, p1 = 2 sigma^2, p2 = 1 / sqrt(2 pi sigma^2), sigma = epsilon / 3):
//   empty_r = sum_s w^2 [t < gt - eps],  near_r = sum_s (w - p2 exp(-(t - gt)^2 / p1))^2 [gt - eps < t < gt + eps]
//   loss = post * mean_r(pre * (mean(empty) + mean(near)) * [gt_r > 0])
// sight (compute_line_of_sight_loss before its ray mask): loss = post * pre * (mean(empty) + mean(near))
// sky, weights based:  loss = post * mean_r(sum_s w^2 * sky_r)
__device__ __forceinline__ float dirac(float t, float gt, float two_sigma_sq, float amp) {
    const float x = t - gt;
    return amp * expf(-(x * x) / two_sigma_sq);
}

__global__ void __launch_bounds__(LOSS_THREADS) ray_loss_fwd_kernel(const LossParams launch) {
    const LossParams p = with_live(launch);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    float sa = 0.0f, sb = 0.0f;
    long long cnt = 0;
    for (int64_t ray = (int64_t)blockIdx.x * LOSS_WARPS + wid; ray < p.n; ray += (int64_t)gridDim.x * LOSS_WARPS) {
        const float* w = p.a + ray * p.s;
        const float gt = __ldg(p.c + ray);
        float e = 0.0f, nr = 0.0f;
        if (p.kind != EMER_RAY_LOSS_SKY_WEIGHTS) {
            const float* t = p.b + ray * p.s;
            const float lo = gt - p.p0, hi = gt + p.p0;
            for (int j = lane; j < p.s; j += 32) {
                const float wj = __ldg(w + j), tj = __ldg(t + j);
                if (tj < lo) e += wj * wj;
                if (tj > lo && tj < hi) {
                    const float d = wj - dirac(tj, gt, p.p1, p.p2);
                    nr += d * d;
                }
            }
            e = warp_sum(e);
            nr = warp_sum(nr);
            if (lane == 0) { sa += e; sb += nr; cnt += gt > 0.0f; }
        } else {
            for (int j = lane; j < p.s; j += 32) {
                const float wj = __ldg(w + j);
                e += wj * wj;
            }
            e = warp_sum(e);
            if (lane == 0) sa += e * gt;
        }
    }
    if (reduce_across_ctas(p.ws, sa, sb, cnt)) {
        const float rays = (float)p.n;
        if (p.kind == EMER_RAY_LOSS_LINE_OF_SIGHT) {
            const float sight = sa / rays + sb / rays;
            const float count = (float)cnt;
            p.out[0] = sight * p.pre * count / rays * p.post;
            p.out[1] = count;
        } else if (p.kind == EMER_RAY_LOSS_SIGHT) {
            p.out[0] = (sa / rays + sb / rays) * p.pre * p.post;
            p.out[1] = rays;
        } else {
            p.out[0] = sa / rays * p.post;
            p.out[1] = rays;
        }
    }
}

__global__ void __launch_bounds__(LOSS_THREADS) ray_loss_bwd_kernel(const LossParams launch) {
    const LossParams p = with_live(launch);
    const float rays = (float)p.n;
    const float g = __ldg(p.g) * p.post / rays;
    // line of sight: every ray's sum enters through mean(empty) + mean(near), scaled by pre and the count of gt > 0
    const float gr = p.kind == EMER_RAY_LOSS_LINE_OF_SIGHT ? g * p.pre * __ldg(p.out + 1) / rays
                                                           : __ldg(p.g) * p.post * p.pre / rays;
    const int64_t total = p.n * p.s;
    for (int64_t i = (int64_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < total; i += (int64_t)gridDim.x * LOSS_THREADS) {
        const int64_t ray = i / p.s;
        const float w = __ldg(p.a + i), gt = __ldg(p.c + ray);
        float d;
        if (p.kind != EMER_RAY_LOSS_SKY_WEIGHTS) {
            const float t = __ldg(p.b + i);
            const float lo = gt - p.p0, hi = gt + p.p0;
            d = 0.0f;
            if (t < lo) d = 2.0f * w * gr;
            if (t > lo && t < hi) d = 2.0f * (w - dirac(t, gt, p.p1, p.p2)) * gr;
        } else {
            d = 2.0f * w * (g * gt);
        }
        p.da[i] = d;
    }
}

// ---------------------------------------------------------------------------------------------- flow cycle loss
// train_emernerf.py:700-740 of the reference, over n rows of 3 (R * S samples):
//   value = coef * (0.5 * mean((f + fpb)^2 + (b + bpf)^2)), the mean over all 3n elements
//   stats = max_row |f|, |b|, |fpb|, |bpf|
// Each input is a [n, 3] view with its own row stride (a column slice of the flow MLP's output rows).
enum { CYC_F = 0, CYC_B = 1, CYC_FPB = 2, CYC_BPF = 3 };

struct CycleParams {
    const float* x[4];       // forward flow, backward flow, forward-predicted backward, backward-predicted forward
    int64_t ld[4];
    int64_t n;
    float coef;
    float* out;              // [6]: value, count, the four maxima in the order of x
    LossWorkspace* ws;
    const float* g;          // backward: upstream gradient (device scalar)
    float* d_fpb;            // backward: [n, 3] contiguous, or null
    float* d_bpf;
};

__device__ __forceinline__ float3 cycle_row(const CycleParams& p, int k, int64_t i) {
    const float* r = p.x[k] + i * p.ld[k];
    return make_float3(__ldg(r), __ldg(r + 1), __ldg(r + 2));
}

// |v| as an unsigned key with the order of the floats: a non-negative float orders as its bits, and clearing the
// sign bit sends every NaN above +inf, so the maximum is NaN when any row is (as torch.max)
__device__ __forceinline__ unsigned int norm_key(float3 v) {
    return __float_as_uint(sqrtf(v.x * v.x + v.y * v.y + v.z * v.z)) & 0x7fffffffu;
}

__device__ __forceinline__ float cycle_term(float f, float p, float b, float q) {
    const float u = f + p, w = b + q;
    return u * u + w * w;
}

__global__ void __launch_bounds__(LOSS_THREADS) cycle_loss_fwd_kernel(const CycleParams p) {
    __shared__ float shf[LOSS_WARPS];
    __shared__ unsigned int shu[LOSS_WARPS];
    float sum = 0.0f;
    unsigned int mx[4] = {0u, 0u, 0u, 0u};
    for (int64_t i = (int64_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * LOSS_THREADS) {
        const float3 f = cycle_row(p, CYC_F, i), b = cycle_row(p, CYC_B, i);
        const float3 fp = cycle_row(p, CYC_FPB, i), bp = cycle_row(p, CYC_BPF, i);
        sum += cycle_term(f.x, fp.x, b.x, bp.x);
        sum += cycle_term(f.y, fp.y, b.y, bp.y);
        sum += cycle_term(f.z, fp.z, b.z, bp.z);
        mx[CYC_F] = max(mx[CYC_F], norm_key(f));
        mx[CYC_B] = max(mx[CYC_B], norm_key(b));
        mx[CYC_FPB] = max(mx[CYC_FPB], norm_key(fp));
        mx[CYC_BPF] = max(mx[CYC_BPF], norm_key(bp));
    }
    sum = block_sum<LOSS_WARPS>(sum, shf);
#pragma unroll
    for (int k = 0; k < 4; ++k) mx[k] = block_max<LOSS_WARPS>(mx[k], shu);
    if (threadIdx.x == 0) {
        p.ws->sum_a[blockIdx.x] = sum;
#pragma unroll
        for (int k = 0; k < 4; ++k) p.ws->norm_max[k][blockIdx.x] = mx[k];
    }
    if (!take_last_ticket(&p.ws->ticket)) return;
    sum = 0.0f;
#pragma unroll
    for (int k = 0; k < 4; ++k) mx[k] = 0u;
    for (int c = threadIdx.x; c < (int)gridDim.x; c += LOSS_THREADS) {
        sum += __ldcg(p.ws->sum_a + c);
#pragma unroll
        for (int k = 0; k < 4; ++k) mx[k] = max(mx[k], __ldcg(p.ws->norm_max[k] + c));
    }
    sum = block_sum<LOSS_WARPS>(sum, shf);
#pragma unroll
    for (int k = 0; k < 4; ++k) mx[k] = block_max<LOSS_WARPS>(mx[k], shu);
    release_ticket(&p.ws->ticket);
    if (threadIdx.x == 0) {
        const float count = (float)(p.n * 3);
        p.out[0] = 0.5f * (sum / count) * p.coef;
        p.out[1] = count;
#pragma unroll
        for (int k = 0; k < 4; ++k) p.out[2 + k] = __uint_as_float(mx[k]);
    }
}

__global__ void __launch_bounds__(LOSS_THREADS) cycle_loss_bwd_kernel(const CycleParams p) {
    const float gs = __ldg(p.g) * p.coef * 0.5f / __ldg(p.out + 1);         // torch's chain: coef, 0.5, the mean
    for (int64_t i = (int64_t)blockIdx.x * LOSS_THREADS + threadIdx.x; i < p.n; i += (int64_t)gridDim.x * LOSS_THREADS) {
        if (p.d_fpb) {
            const float3 f = cycle_row(p, CYC_F, i), fp = cycle_row(p, CYC_FPB, i);
            float* d = p.d_fpb + i * 3;
            d[0] = 2.0f * (f.x + fp.x) * gs;
            d[1] = 2.0f * (f.y + fp.y) * gs;
            d[2] = 2.0f * (f.z + fp.z) * gs;
        }
        if (p.d_bpf) {
            const float3 b = cycle_row(p, CYC_B, i), bp = cycle_row(p, CYC_BPF, i);
            float* d = p.d_bpf + i * 3;
            d[0] = 2.0f * (b.x + bp.x) * gs;
            d[1] = 2.0f * (b.y + bp.y) * gs;
            d[2] = 2.0f * (b.z + bp.z) * gs;
        }
    }
}

// persistent grid: at most two CTAs per SM (and the workspace's LOSS_MAX_CTAS partials)
static int loss_grid(int64_t work_items, int per_cta) {
    int64_t blocks = ceil_div(work_items, per_cta);
    int64_t cap = (int64_t)sm_count() * 2;
    if (cap > LOSS_MAX_CTAS) cap = LOSS_MAX_CTAS;
    if (blocks > cap) blocks = cap;
    return blocks < 1 ? 1 : (int)blocks;
}

}  // namespace emer

using namespace emer;

extern "C" int emer_pointwise_loss_fwd(int kind, const float* a, const float* b, int64_t n, float p0, float p1,
                                       float pre, float post, float* out, void* workspace, void* stream) {
    EMER_REQUIRE(kind >= EMER_LOSS_L1 && kind <= EMER_LOSS_ENTROPY, "emer_pointwise_loss_fwd: unknown kind %d", kind);
    EMER_REQUIRE(a && out && workspace && (kind == EMER_LOSS_SPARSITY || b), "emer_pointwise_loss_fwd: NULL pointer");
    EMER_REQUIRE(n >= 0, "emer_pointwise_loss_fwd: negative size");
    LossParams p{kind, a, b, nullptr, n, 0, p0, p1, 0.0f, pre, post, out, (LossWorkspace*)workspace, nullptr, nullptr,
                 nullptr};
    pointwise_loss_fwd_kernel<<<loss_grid(n, LOSS_THREADS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_pointwise_loss_fwd");
}

extern "C" int emer_pointwise_loss_bwd(int kind, const float* a, const float* b, int64_t n, float p0, float p1,
                                       float pre, float post, const float* fwd_out, const float* g, float* da, float* db,
                                       void* stream) {
    EMER_REQUIRE(kind >= EMER_LOSS_L1 && kind <= EMER_LOSS_ENTROPY, "emer_pointwise_loss_bwd: unknown kind %d", kind);
    EMER_REQUIRE(a && fwd_out && g && (kind == EMER_LOSS_SPARSITY || b), "emer_pointwise_loss_bwd: NULL pointer");
    EMER_REQUIRE(da || (kind == EMER_LOSS_ENTROPY && db), "emer_pointwise_loss_bwd: no gradient requested");
    if (n <= 0) return 0;
    LossParams p{kind, a, b, nullptr, n, 0, p0, p1, 0.0f, pre, post, (float*)fwd_out, nullptr, g, da, db};
    pointwise_loss_bwd_kernel<<<loss_grid(n, LOSS_THREADS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_pointwise_loss_bwd");
}

extern "C" int emer_ray_loss_fwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays,
                                 int n_samples, float eps, float two_sigma_sq, float amp, float pre, float post, float* out,
                                 void* workspace, void* stream) {
    EMER_REQUIRE(kind >= EMER_RAY_LOSS_LINE_OF_SIGHT && kind <= EMER_RAY_LOSS_SIGHT, "emer_ray_loss_fwd: unknown kind %d", kind);
    EMER_REQUIRE(w && gt && out && workspace && (kind == EMER_RAY_LOSS_SKY_WEIGHTS || t),
                 "emer_ray_loss_fwd: NULL pointer");
    EMER_REQUIRE(n_rays >= 0 && n_samples >= 1, "emer_ray_loss_fwd: bad shape");
    LossParams p{kind, w, t, gt, n_rays, n_samples, eps, two_sigma_sq, amp, pre, post, out, (LossWorkspace*)workspace,
                 nullptr, nullptr, nullptr};
    ray_loss_fwd_kernel<<<loss_grid(n_rays, LOSS_WARPS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_ray_loss_fwd");
}

extern "C" int emer_ray_loss_bwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays,
                                 int n_samples, float eps, float two_sigma_sq, float amp, float pre, float post,
                                 const float* fwd_out, const float* g, float* dw, void* stream) {
    EMER_REQUIRE(kind >= EMER_RAY_LOSS_LINE_OF_SIGHT && kind <= EMER_RAY_LOSS_SIGHT, "emer_ray_loss_bwd: unknown kind %d", kind);
    EMER_REQUIRE(w && gt && fwd_out && g && dw && (kind == EMER_RAY_LOSS_SKY_WEIGHTS || t),
                 "emer_ray_loss_bwd: NULL pointer");
    EMER_REQUIRE(n_rays >= 0 && n_samples >= 1, "emer_ray_loss_bwd: bad shape");
    if (n_rays == 0) return 0;
    LossParams p{kind, w, t, gt, n_rays, n_samples, eps, two_sigma_sq, amp, pre, post, (float*)fwd_out, nullptr, g, dw,
                 nullptr};
    ray_loss_bwd_kernel<<<loss_grid(n_rays * n_samples, LOSS_THREADS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_ray_loss_bwd");
}

extern "C" int emer_ray_loss_live_fwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays,
                                      int n_samples, const float* consts, float post, float* out, void* workspace,
                                      void* stream) {
    EMER_REQUIRE(kind == EMER_RAY_LOSS_LINE_OF_SIGHT || kind == EMER_RAY_LOSS_SIGHT,
                 "emer_ray_loss_live_fwd: kind %d has no live constants", kind);
    EMER_REQUIRE(w && t && gt && consts && out && workspace, "emer_ray_loss_live_fwd: NULL pointer");
    EMER_REQUIRE(n_rays >= 0 && n_samples >= 1, "emer_ray_loss_live_fwd: bad shape");
    LossParams p{kind, w, t, gt, n_rays, n_samples, 0.0f, 0.0f, 0.0f, 0.0f, post, out, (LossWorkspace*)workspace,
                 nullptr, nullptr, nullptr, consts};
    ray_loss_fwd_kernel<<<loss_grid(n_rays, LOSS_WARPS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_ray_loss_live_fwd");
}

extern "C" int emer_ray_loss_live_bwd(int kind, const float* w, const float* t, const float* gt, int64_t n_rays,
                                      int n_samples, const float* consts, float post, const float* fwd_out,
                                      const float* g, float* dw, void* stream) {
    EMER_REQUIRE(kind == EMER_RAY_LOSS_LINE_OF_SIGHT || kind == EMER_RAY_LOSS_SIGHT,
                 "emer_ray_loss_live_bwd: kind %d has no live constants", kind);
    EMER_REQUIRE(w && t && gt && consts && fwd_out && g && dw, "emer_ray_loss_live_bwd: NULL pointer");
    EMER_REQUIRE(n_rays >= 0 && n_samples >= 1, "emer_ray_loss_live_bwd: bad shape");
    if (n_rays == 0) return 0;
    LossParams p{kind, w, t, gt, n_rays, n_samples, 0.0f, 0.0f, 0.0f, 0.0f, post, (float*)fwd_out, nullptr, g, dw,
                 nullptr, consts};
    ray_loss_bwd_kernel<<<loss_grid(n_rays * n_samples, LOSS_THREADS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_ray_loss_live_bwd");
}

static CycleParams cycle_params(const float* f, int64_t ld_f, const float* b, int64_t ld_b, const float* fpb,
                                int64_t ld_fpb, const float* bpf, int64_t ld_bpf, int64_t n, float coef) {
    CycleParams p{};
    p.x[CYC_F] = f; p.x[CYC_B] = b; p.x[CYC_FPB] = fpb; p.x[CYC_BPF] = bpf;
    p.ld[CYC_F] = ld_f; p.ld[CYC_B] = ld_b; p.ld[CYC_FPB] = ld_fpb; p.ld[CYC_BPF] = ld_bpf;
    p.n = n;
    p.coef = coef;
    return p;
}

extern "C" int emer_cycle_loss_fwd(const float* f, int64_t ld_f, const float* b, int64_t ld_b, const float* fpb,
                                   int64_t ld_fpb, const float* bpf, int64_t ld_bpf, int64_t n, float coef, float* out,
                                   void* workspace, void* stream) {
    EMER_REQUIRE(f && b && fpb && bpf && out && workspace, "emer_cycle_loss_fwd: NULL pointer");
    EMER_REQUIRE(n >= 1, "emer_cycle_loss_fwd: no rows");        // the maxima of nothing are undefined
    EMER_REQUIRE(ld_f >= 3 && ld_b >= 3 && ld_fpb >= 3 && ld_bpf >= 3, "emer_cycle_loss_fwd: row stride below 3");
    CycleParams p = cycle_params(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, coef);
    p.out = out;
    p.ws = (LossWorkspace*)workspace;
    cycle_loss_fwd_kernel<<<loss_grid(n, LOSS_THREADS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_cycle_loss_fwd");
}

extern "C" int emer_cycle_loss_bwd(const float* f, int64_t ld_f, const float* b, int64_t ld_b, const float* fpb,
                                   int64_t ld_fpb, const float* bpf, int64_t ld_bpf, int64_t n, float coef,
                                   const float* fwd_out, const float* g, float* d_fpb, float* d_bpf, void* stream) {
    EMER_REQUIRE(f && b && fpb && bpf && fwd_out && g, "emer_cycle_loss_bwd: NULL pointer");
    EMER_REQUIRE(d_fpb || d_bpf, "emer_cycle_loss_bwd: no gradient requested");
    EMER_REQUIRE(n >= 1, "emer_cycle_loss_bwd: no rows");
    EMER_REQUIRE(ld_f >= 3 && ld_b >= 3 && ld_fpb >= 3 && ld_bpf >= 3, "emer_cycle_loss_bwd: row stride below 3");
    CycleParams p = cycle_params(f, ld_f, b, ld_b, fpb, ld_fpb, bpf, ld_bpf, n, coef);
    p.out = (float*)fwd_out;
    p.g = g;
    p.d_fpb = d_fpb;
    p.d_bpf = d_bpf;
    cycle_loss_bwd_kernel<<<loss_grid(n, LOSS_THREADS), LOSS_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch("emer_cycle_loss_bwd");
}
