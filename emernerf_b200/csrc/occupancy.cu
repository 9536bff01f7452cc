// The few-shot occupancy evaluation of the reference (datasets/metrics.py:249-472: collect_centroids and
// eval_few_shot_occ with knn_predict(knn_k=1, similarity="cosine")), one launch per chunk of voxels.  The reference
// keeps the voxels with density > 0.2 by boolean indexing (a host sync), runs the field a second time on them for the
// features, concatenates every kept feature row of every train frame before it takes per-class means, and reads each
// per-class count with .item().  Here the filter, the per-class sums and the classification read the rows of a single
// field pass in place and add into caller-owned device buffers, so any number of frames and chunks add up without a
// sync.
//
// emer_occ_accumulate: one warp per row (lanes over 16-byte column groups) adds each kept row into the warp's own fp64
// [classes, channels] accumulator in shared memory; rows reach a warp in a fixed order, so no atomics are needed.
// emer_occ_classify: one thread per row; every warp stages 32 rows x 32 columns at a time in shared memory and scores
// its row against every normalised centroid in fp64.
//
// Reduction: per-CTA records go to the caller's workspace, and the CTA that takes the last ticket adds them in CTA
// order into the caller's buffers and resets the ticket.  No float atomics: the same inputs on the same device give
// bit-identical results.
#include <math.h>

#include "common.cuh"
#include "cta_reduce.cuh"

namespace emer {

constexpr int OCC_THREADS = 256;
constexpr int OCC_MAX_CTAS = 256;
constexpr int OCC_MAX_C = EMER_OCC_MAX_CHANNELS;
constexpr int OCC_MAX_K = EMER_OCC_MAX_CLASSES;
constexpr int OCC_UNROLL = 4;                       // rows in flight per warp (accumulate)
constexpr int OCC_TILE = 32;                        // rows x columns staged per warp (classify)
constexpr int OCC_TILE_LD = OCC_TILE + 1;           // padded: the staging stores and the row reads are conflict-free
constexpr size_t OCC_WS_HEADER = 256;               // ticket, then the per-CTA records
constexpr size_t OCC_SMEM_BUDGET = 192 * 1024;      // dynamic shared memory of one accumulate CTA at most
static_assert(OCC_WS_HEADER + (size_t)OCC_MAX_CTAS * (OCC_MAX_K * OCC_MAX_C + 2 * OCC_MAX_K + 2) * 8 <=
                  EMER_OCC_WORKSPACE_BYTES,
              "workspace layout exceeds the ABI size");

struct OccParams {
    const float* feat;          // n rows of c floats, row stride ld_feat
    int64_t ld_feat;
    int c;
    const float* density;       // n values, stride ld_density
    int64_t ld_density;
    const int64_t* labels;      // n
    int64_t n;
    int k;
    float threshold;
    const float* centroids;     // [k, c] (classify)
    const int64_t* label_bank;  // [k]    (classify)
    double* sums;               // [k, c] (accumulate)
    int64_t* counts;
    unsigned char* ws;
};

// Publishes this CTA's record (nd doubles and ni counters, in shared memory); the CTA that takes the last ticket adds
// the records of all CTAs, in CTA order, into out_d / out_i and resets the ticket.
__device__ void occ_finish(const double* sd, int nd, const unsigned long long* si, int ni, double* out_d,
                           int64_t* out_i, unsigned char* ws) {
    unsigned int* ticket = (unsigned int*)ws;
    double* pd = (double*)(ws + OCC_WS_HEADER);
    long long* pi = (long long*)(pd + (size_t)gridDim.x * nd);
    for (int i = threadIdx.x; i < nd; i += blockDim.x) pd[(size_t)blockIdx.x * nd + i] = sd[i];
    for (int i = threadIdx.x; i < ni; i += blockDim.x) pi[(size_t)blockIdx.x * ni + i] = (long long)si[i];
    if (!take_last_ticket(ticket)) return;
    for (int i = threadIdx.x; i < nd; i += blockDim.x) {
        double s = 0.0;
        for (int b = 0; b < (int)gridDim.x; ++b) s += __ldcg(pd + (size_t)b * nd + i);
        out_d[i] += s;
    }
    for (int i = threadIdx.x; i < ni; i += blockDim.x) {
        long long s = 0;
        for (int b = 0; b < (int)gridDim.x; ++b) s += __ldcg(pi + (size_t)b * ni + i);
        out_i[i] += s;
    }
    release_ticket(ticket);
}

// class of row r if it passes the filter (density > threshold, NaN fails; 0 <= label < k), else -1
__device__ __forceinline__ int occ_class(const OccParams& p, int64_t r) {
    const float d = __ldg(p.density + r * p.ld_density);
    const long long l = __ldg((const long long*)p.labels + r);
    return (d > p.threshold && l >= 0 && l < p.k) ? (int)l : -1;
}

// ---------------------------------------------------------------------------------------------- per-class sums
__global__ void __launch_bounds__(OCC_THREADS) occ_accumulate_kernel(const OccParams p) {
    extern __shared__ double acc[];                   // [warps][k * c]
    __shared__ unsigned long long cnt[OCC_MAX_K];
    const int warps = blockDim.x >> 5, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int kc = p.k * p.c, c4 = p.c >> 2;
    for (int i = threadIdx.x; i < warps * kc; i += blockDim.x) acc[i] = 0.0;
    if (threadIdx.x < OCC_MAX_K) cnt[threadIdx.x] = 0ull;
    __syncthreads();
    double* mine = acc + (size_t)wid * kc;
    const int64_t nw = (int64_t)gridDim.x * warps;
    for (int64_t r0 = (int64_t)blockIdx.x * warps + wid; r0 < p.n; r0 += OCC_UNROLL * nw) {
        int cls[OCC_UNROLL];
        float4 v[OCC_UNROLL][2];
#pragma unroll
        for (int u = 0; u < OCC_UNROLL; ++u) {
            const int64_t r = r0 + u * nw;
            cls[u] = r < p.n ? occ_class(p, r) : -1;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = lane + 32 * h;
                v[u][h] = (cls[u] >= 0 && j < c4) ? __ldg((const float4*)(p.feat + r * p.ld_feat) + j)
                                                  : make_float4(0.f, 0.f, 0.f, 0.f);
            }
        }
#pragma unroll
        for (int u = 0; u < OCC_UNROLL; ++u) {
            if (cls[u] < 0) continue;
            if (lane == 0) atomicAdd(&cnt[cls[u]], 1ull);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = lane + 32 * h;
                if (j >= c4) continue;
                double* a = mine + (size_t)cls[u] * p.c + 4 * j;
                a[0] += (double)v[u][h].x;
                a[1] += (double)v[u][h].y;
                a[2] += (double)v[u][h].z;
                a[3] += (double)v[u][h].w;
            }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < kc; i += blockDim.x) {
        double s = acc[i];
        for (int w = 1; w < warps; ++w) s += acc[(size_t)w * kc + i];
        acc[i] = s;
    }
    __syncthreads();
    occ_finish(acc, kc, cnt, p.k, p.sums, p.counts, p.ws);
}

// ---------------------------------------------------------------------------------------------- classification
// counts: [0, k) totals per class, [k, 2k) correct per class, 2k measured (density > threshold), 2k+1 labels out of
// range among the measured
template <int MAXK>
__device__ __forceinline__ void occ_classify(const OccParams& p) {
    extern __shared__ double chat[];                  // [c][MAXK] normalised centroids (0 for j >= k), then the tiles
    __shared__ unsigned long long cnt[2 * OCC_MAX_K + 2];
    const int warps = blockDim.x >> 5, lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int C = p.c, K = p.k;
    float* tile = (float*)(chat + (size_t)C * MAXK) + (size_t)wid * OCC_TILE * OCC_TILE_LD;
    for (int j = wid; j < MAXK; j += warps) {
        double ss = 0.0;
        if (j < K)
            for (int c = lane; c < C; c += 32) {
                const double v = __ldg(p.centroids + (size_t)j * C + c);
                ss = fma(v, v, ss);
            }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
        const double den = sqrt(ss) + 1e-7;
        for (int c = lane; c < C; c += 32)
            chat[(size_t)c * MAXK + j] = j < K ? (double)__ldg(p.centroids + (size_t)j * C + c) / den : 0.0;
    }
    if (threadIdx.x < 2 * OCC_MAX_K + 2) cnt[threadIdx.x] = 0ull;
    __syncthreads();
    const int sub = lane >> 3, q = lane & 7;          // staging: 4 rows x 8 float4 per load
    const int64_t stride = (int64_t)gridDim.x * warps * OCC_TILE;
    for (int64_t base = ((int64_t)blockIdx.x * warps + wid) * OCC_TILE; base < p.n; base += stride) {
        const int64_t r = base + lane;
        bool keep = false;
        long long lab = -1;
        if (r < p.n) {
            keep = __ldg(p.density + r * p.ld_density) > p.threshold;
            lab = __ldg((const long long*)p.labels + r);
        }
        const bool ok = keep && lab >= 0 && lab < K;
        if (keep) {
            atomicAdd(&cnt[2 * K], 1ull);
            if (!ok) atomicAdd(&cnt[2 * K + 1], 1ull);
        }
        const unsigned okm = __ballot_sync(0xffffffffu, ok);
        if (okm == 0u) continue;
        double acc[MAXK];
#pragma unroll
        for (int j = 0; j < MAXK; ++j) acc[j] = 0.0;
        for (int c0 = 0; c0 < C; c0 += OCC_TILE) {
            float4 v[OCC_TILE / 4];
#pragma unroll
            for (int i = 0; i < OCC_TILE / 4; ++i) {
                const int row = 4 * i + sub, col = c0 + 4 * q;
                v[i] = ((okm >> row) & 1u) && col < C
                           ? __ldg((const float4*)(p.feat + (base + row) * p.ld_feat + col))
                           : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int i = 0; i < OCC_TILE / 4; ++i) {
                float* t = tile + (4 * i + sub) * OCC_TILE_LD + 4 * q;
                t[0] = v[i].x; t[1] = v[i].y; t[2] = v[i].z; t[3] = v[i].w;
            }
            __syncwarp();
            const int cn = min(OCC_TILE, C - c0);
            for (int c = 0; c < cn; ++c) {
                const double x = tile[lane * OCC_TILE_LD + c];
                const double2* w = (const double2*)(chat + (size_t)(c0 + c) * MAXK);
#pragma unroll
                for (int j = 0; j < MAXK / 2; ++j) {
                    const double2 h = w[j];
                    acc[2 * j] = fma(x, h.x, acc[2 * j]);
                    acc[2 * j + 1] = fma(x, h.y, acc[2 * j + 1]);
                }
            }
            __syncwarp();                             // the tile is read before the next columns overwrite it
        }
        if (!ok) continue;
        int best = 0;
        double top = acc[0];
#pragma unroll
        for (int j = 1; j < MAXK; ++j)
            if (j < K && acc[j] > top) {             // strict: an exact tie keeps the lower index
                top = acc[j];
                best = j;
            }
        atomicAdd(&cnt[lab], 1ull);
        if (__ldg((const long long*)p.label_bank + best) == lab) atomicAdd(&cnt[K + lab], 1ull);
    }
    __syncthreads();
    occ_finish(nullptr, 0, cnt, 2 * K + 2, nullptr, p.counts, p.ws);
}

// one kernel per class bound: the scores live in registers, so their count is a compile-time constant
__global__ void __launch_bounds__(OCC_THREADS) occ_classify16_kernel(const OccParams p) { occ_classify<16>(p); }
__global__ void __launch_bounds__(OCC_THREADS) occ_classify32_kernel(const OccParams p) { occ_classify<32>(p); }

static int occ_grid(int64_t rows_per_cta, int64_t n) {
    int64_t blocks = ceil_div(n, rows_per_cta);
    int64_t cap = (int64_t)sm_count() * 2;
    if (cap > OCC_MAX_CTAS) cap = OCC_MAX_CTAS;
    if (blocks > cap) blocks = cap;
    return blocks < 1 ? 1 : (int)blocks;
}

static int occ_check(const char* what, const float* feat, int64_t ld_feat, int channels, const float* density,
                     int64_t ld_density, const int64_t* labels, int64_t n, int n_classes, const void* counts,
                     const void* workspace) {
    EMER_REQUIRE(feat && density && labels && counts && workspace, "%s: NULL pointer", what);
    EMER_REQUIRE(n >= 0, "%s: negative size", what);
    EMER_REQUIRE(channels >= 4 && channels <= OCC_MAX_C && channels % 4 == 0,
                 "%s: %d channels (a multiple of 4, at most %d)", what, channels, OCC_MAX_C);
    EMER_REQUIRE(n_classes >= 1 && n_classes <= OCC_MAX_K, "%s: %d classes (1..%d)", what, n_classes, OCC_MAX_K);
    EMER_REQUIRE(ld_feat >= channels && ld_feat % 4 == 0 && (uintptr_t)feat % 16 == 0,
                 "%s: feature rows must be 16-byte aligned (row stride %lld)", what, (long long)ld_feat);
    EMER_REQUIRE(ld_density >= 1, "%s: density stride %lld", what, (long long)ld_density);
    return 0;
}

}  // namespace emer

using namespace emer;

extern "C" int emer_occ_accumulate(const float* feat, int64_t ld_feat, int channels, const float* density,
                                   int64_t ld_density, const int64_t* labels, int64_t n, int n_classes,
                                   float threshold, double* sums, int64_t* counts, void* workspace, void* stream) {
    const int rc = occ_check("emer_occ_accumulate", feat, ld_feat, channels, density, ld_density, labels, n,
                             n_classes, counts, workspace);
    if (rc) return rc;
    EMER_REQUIRE(sums, "emer_occ_accumulate: NULL pointer");
    const size_t per_warp = (size_t)n_classes * channels * sizeof(double);
    int warps = (int)(OCC_SMEM_BUDGET / per_warp);
    warps = warps < 1 ? 1 : (warps > OCC_THREADS / 32 ? OCC_THREADS / 32 : warps);
    const size_t smem = per_warp * warps;
    cudaFuncSetAttribute(occ_accumulate_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    OccParams p{};
    p.feat = feat; p.ld_feat = ld_feat; p.c = channels;
    p.density = density; p.ld_density = ld_density; p.labels = labels; p.n = n; p.k = n_classes;
    p.threshold = threshold; p.sums = sums; p.counts = counts; p.ws = (unsigned char*)workspace;
    occ_accumulate_kernel<<<occ_grid((int64_t)warps * OCC_UNROLL * 8, n), warps * 32, smem, (cudaStream_t)stream>>>(p);
    return check_launch("emer_occ_accumulate");
}

static void occ_classify_launch(void (*kernel)(const OccParams), int maxk, const OccParams& p, cudaStream_t stream) {
    const size_t smem = (size_t)p.c * maxk * sizeof(double) +
                        (size_t)(OCC_THREADS / 32) * OCC_TILE * OCC_TILE_LD * sizeof(float);
    cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    kernel<<<occ_grid(OCC_THREADS * 4, p.n), OCC_THREADS, smem, stream>>>(p);
}

extern "C" int emer_occ_classify(const float* feat, int64_t ld_feat, int channels, const float* density,
                                 int64_t ld_density, const int64_t* labels, int64_t n, const float* centroids,
                                 int n_classes, const int64_t* label_bank, float threshold, int64_t* counts,
                                 void* workspace, void* stream) {
    const int rc = occ_check("emer_occ_classify", feat, ld_feat, channels, density, ld_density, labels, n,
                             n_classes, counts, workspace);
    if (rc) return rc;
    EMER_REQUIRE(centroids && label_bank, "emer_occ_classify: NULL pointer");
    OccParams p{};
    p.feat = feat; p.ld_feat = ld_feat; p.c = channels;
    p.density = density; p.ld_density = ld_density; p.labels = labels; p.n = n; p.k = n_classes;
    p.threshold = threshold; p.centroids = centroids; p.label_bank = label_bank; p.counts = counts;
    p.ws = (unsigned char*)workspace;
    if (n_classes <= 16) occ_classify_launch(occ_classify16_kernel, 16, p, (cudaStream_t)stream);
    else occ_classify_launch(occ_classify32_kernel, 32, p, (cudaStream_t)stream);
    return check_launch("emer_occ_classify");
}
