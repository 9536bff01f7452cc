// Weight gradients  dW[n_out, k] += dZ^T X,  db += column sums of dZ,  on Hopper warpgroup MMA (3xTF32, tc_common.cuh).
// Entry points: emer_linear_tc_bwd_weight (any n_out <= 128, k <= 256) and emer_linear_tc_bwd_weight_mn (the 64-wide
// layers of the field chain, read as they lie in memory: row-major X and dZ); both run wgrad_kernel.
// D[k x n_out] = X^T dZ: A = X^T straight from the row-major X (the 8 lanes with the same q read one 32-byte sector of
// a row), B = dZ^T staged per tile into K-major panels; D stays in registers across the persistent CTA's tiles and is
// flushed once with atomics (DESIGN.md §5.3).  HBM-bound: (k + n_out) * 4 B per row.
#include "common.cuh"
#include "tc_common.cuh"

namespace emer {
namespace wg {

using namespace emer::tc;

constexpr int TR = 32;                       // rows per tile = 4 k steps
constexpr int MIN_TILES = 4;

struct Params {
    const float* x; int64_t ldx; int k;       // [n, ldx]
    const float* dz; int64_t lddz; int n_out; // [n, lddz]
    float* dw;                                // [n_out, k] row-major, accumulated
    float* db;                                // [n_out] accumulated, or null
    int64_t n;
};

// NP: n_out padded to a power of two in [16, 128], so that every thread stages one fixed column (blockDim % NP == 0);
// MB: warpgroups = 64-feature blocks of X in the CTA
template <int NP, int MB>
__global__ void __launch_bounds__(128 * MB) wgrad_kernel(const Params p) {
    constexpr int NT = 128 * MB, PER = (TR * NP + NT - 1) / NT;      // dZ values a thread stages per tile (at most)
    __shared__ __align__(128) uint8_t smem[2 * TR * NP * 4];
    uint8_t* b_hi = smem;
    uint8_t* b_lo = smem + TR * NP * 4;
    const int tid = threadIdx.x;
    const int wgi = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
    const int f0 = wgi * 64 + 16 * w + (lane >> 2), f1 = f0 + 8;    // this thread's two features (A rows)
    const bool fok0 = f0 < p.k, fok1 = f1 < p.k;
    const int o_st = tid % NP;                                       // the column this thread stages
    const uint32_t bh = smem_u32(b_hi), bl = smem_u32(b_lo);
    const int64_t n_tiles = (p.n + TR - 1) / TR;

    float xr[TR / 8][4], zr[PER];
    auto load = [&](int64_t tile) {
        const int64_t r_base = tile * TR;
#pragma unroll
        for (int ks = 0; ks < TR / 8; ++ks) {
            const int64_t ra = r_base + 8 * ks + 2 * q, rb = ra + 1;
            const bool oka = ra < p.n, okb = rb < p.n;
            xr[ks][0] = (oka && fok0) ? __ldg(p.x + ra * p.ldx + f0) : 0.0f;
            xr[ks][1] = (okb && fok0) ? __ldg(p.x + rb * p.ldx + f0) : 0.0f;
            xr[ks][2] = (oka && fok1) ? __ldg(p.x + ra * p.ldx + f1) : 0.0f;
            xr[ks][3] = (okb && fok1) ? __ldg(p.x + rb * p.ldx + f1) : 0.0f;
        }
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            const int e = tid + i * NT;                                  // (o_st, e / NP) of the tile
            const int64_t row = r_base + e / NP;
            zr[i] = (e < TR * NP && row < p.n && o_st < p.n_out) ? __ldg(p.dz + row * p.lddz + o_st) : 0.0f;
        }
    };

    float acc[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) acc[i] = 0.0f;
    float dbp = 0.0f;
    load(blockIdx.x);
    for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        __syncthreads();                      // the previous tile's MMAs have finished reading B
#pragma unroll
        for (int i = 0; i < PER; ++i) {
            const int e = tid + i * NT;
            if (e < TR * NP) {
                dbp += zr[i];
                float h, l;
                split(zr[i], h, l);
                const int off = b_off(o_st, e / NP, NP);
                *reinterpret_cast<float*>(b_hi + off) = h;
                *reinterpret_cast<float*>(b_lo + off) = l;
            }
        }
        fence_async_proxy();
        __syncthreads();
        uint32_t ahi[TR / 8][4], alo[TR / 8][4];
#pragma unroll
        for (int ks = 0; ks < TR / 8; ++ks) frag_split(xr[ks][0], xr[ks][1], xr[ks][2], xr[ks][3], ahi[ks], alo[ks]);
        load(tile + gridDim.x);               // the next tile's values arrive under this tile's MMAs
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < TR / 8; ++ks) mma3<NP>(acc, ahi[ks], alo[ks], b_desc(bh, NP, ks, 0), b_desc(bl, NP, ks, 0), 1);
        wg_commit();
        wg_wait0();
    }
    // flush: D[f][o] -> dW[o, f]
#pragma unroll
    for (int j = 0; j < NP / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int f = e < 2 ? f0 : f1, o = 8 * j + 2 * q + (e & 1);
            if ((e < 2 ? fok0 : fok1) && o < p.n_out) atomicAdd(p.dw + (int64_t)o * p.k + f, acc[4 * j + e]);
        }
    }
    if (p.db && o_st < p.n_out) atomicAdd(p.db + o_st, dbp);
}

template <int NP, int MB>
static int launch_t(const Params& p, cudaStream_t st, const char* what) {
    // persistent grid of the CTAs resident at once, with at least MIN_TILES tiles each (every CTA ends with k x n_out
    // atomics onto the same dW addresses, which would dominate small products such as the 8192-row per-ray ones)
    static int cache[64] = {0};
    int64_t grid = (int64_t)sm_count() * resident_ctas(wgrad_kernel<NP, MB>, 128 * MB, 0, st, cache);
    const int64_t ctas = ceil_div(ceil_div(p.n, TR), MIN_TILES);
    if (grid > ctas) grid = ctas;
    wgrad_kernel<NP, MB><<<(unsigned)grid, 128 * MB, 0, st>>>(p);
    return check_launch(what);
}

template <int NP>
static int launch_np(const Params& p, cudaStream_t st, const char* what) {
    switch ((p.k + 63) / 64) {
        case 1: return launch_t<NP, 1>(p, st, what);
        case 2: return launch_t<NP, 2>(p, st, what);
        case 3: return launch_t<NP, 3>(p, st, what);
        default: return launch_t<NP, 4>(p, st, what);
    }
}

static int launch(const Params& p, cudaStream_t st, const char* what) {
    if (p.n_out <= 16) return launch_np<16>(p, st, what);
    if (p.n_out <= 32) return launch_np<32>(p, st, what);
    if (p.n_out <= 64) return launch_np<64>(p, st, what);
    return launch_np<128>(p, st, what);
}

}  // namespace wg
}  // namespace emer

extern "C" int emer_linear_tc_bwd_weight(const float* x, int64_t ldx, const float* dz, int64_t lddz, float* dw,
                                         float* db, int64_t n, int k, int n_out, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && dz && dw, "emer_linear_tc_bwd_weight: NULL pointer");
    EMER_REQUIRE(n_out <= 128 && k <= 256, "emer_linear_tc_bwd_weight: widths k=%d n_out=%d out of range", k, n_out);
    EMER_REQUIRE(ldx % 4 == 0 && lddz % 4 == 0 && ((uintptr_t)x & 15) == 0 && ((uintptr_t)dz & 15) == 0,
                 "emer_linear_tc_bwd_weight: rows must be 16-byte aligned (ldx=%lld lddz=%lld)", (long long)ldx,
                 (long long)lddz);
    EMER_REQUIRE((k + 3) / 4 * 4 <= ldx, "emer_linear_tc_bwd_weight: row stride %lld shorter than padded width %d",
                 (long long)ldx, (k + 3) / 4 * 4);
    EMER_REQUIRE((n_out + 3) / 4 * 4 <= lddz, "emer_linear_tc_bwd_weight: dZ rows too short");
    emer::wg::Params p{x, ldx, k, dz, lddz, n_out, dw, db, n};
    return emer::wg::launch(p, (cudaStream_t)stream, "emer_linear_tc_bwd_weight");
}

extern "C" int emer_linear_tc_bwd_weight_mn(const float* x, int64_t ldx, const float* dz, int64_t lddz, float* dw, float* db,
                                            int64_t n, int k, int n_out, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && dz && dw, "emer_linear_tc_bwd_weight_mn: NULL pointer");
    EMER_REQUIRE(n_out == 64 && k >= 4 && k <= 128, "emer_linear_tc_bwd_weight_mn: shape k=%d n_out=%d (need n_out = 64, k <= 128)", k, n_out);
    EMER_REQUIRE(ldx % 4 == 0 && lddz % 4 == 0 && ((uintptr_t)x & 15) == 0 && ((uintptr_t)dz & 15) == 0 && (k + 3) / 4 * 4 <= ldx,
                 "emer_linear_tc_bwd_weight_mn: rows must be 16-byte aligned");
    emer::wg::Params p{x, ldx, k, dz, lddz, n_out, dw, db, n};
    return emer::wg::launch(p, (cudaStream_t)stream, "emer_linear_tc_bwd_weight_mn");
}
