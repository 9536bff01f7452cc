// The fused field chain's weight gradients in one persistent pass (emer_field_wgrad).  Every row buffer that
// field_bwd_kernel leaves in HBM is read once, and the five products dW += dZ^T X of the chain's layers accumulate in
// registers with the 3xTF32 warpgroup MMA of tc_common.cuh (the arithmetic of wgrad_mn.cu, summed in another order).
//
// Per 16-row tile, cp.async copies enc, hb, hg = [h0 | geo], h1, dz1, d1 = [dZ0 | dF], dzb, d_sem and dz2 into a
// STAGES-deep shared-memory ring, so tiles t+1 .. t+STAGES-1 are in flight while tile t is computed.  Every dZ column
// is split once into K-major hi / lo panels (the B operands, shared by the products that use them) and summed into its
// bias; each warpgroup reads its X^T fragments (the A operands) out of the landed tile:
//   warpgroup 0:  enc x dzb -> dWb0,  hb x dF -> dWb1[:64]
//   warpgroup 1:  geo x dZ0 -> dW0g,  geo x dz1 -> dW1g,  h1 x dz2 -> dW2
//   warpgroup 2:  h0 x dz1 -> dW1h,   hb x d_sem -> dWb1[64:]
// The accumulators stay in registers across the CTA's tiles and are flushed once with atomics (DESIGN.md §5.3).
// HBM-bound: (k_enc + 64 + 128 + 64 + 3 + 64 + 128 + 64 [+ 64 with d_sem]) * 4 B per row.
#include "common.cuh"
#include "tc_common.cuh"

namespace emer {
namespace fw {

using namespace emer::tc;

constexpr int TR = 16;               // rows per tile = 2 k steps
constexpr int STAGES = 4;            // ring depth
constexpr int THREADS = 384;         // three warpgroups
constexpr int MIN_TILES = 4;         // per CTA: each CTA ends with ~25 K atomics onto the same addresses

// B panels (hi, then lo right behind it) of one tile: TR rows of 64 (dz2: 8) columns
constexpr int PANEL64 = TR * 64 * 4, PANEL8 = TR * 8 * 4;
constexpr int P_DZB = 0, P_DF = 2 * PANEL64, P_DSEM = 4 * PANEL64, P_DZ0 = 6 * PANEL64, P_DZ1 = 8 * PANEL64,
              P_DZ2 = 10 * PANEL64, P_BYTES = P_DZ2 + 2 * PANEL8;

// float offsets inside one ring stage.  Rows are padded by 4 floats, a row stride of 4 (mod 32) banks: the A-fragment
// reads (8 features x 4 rows per warp) are conflict-free.  Without the colour head (HEAD = false) only the dF half of
// d1 is loaded, and hg, h1, dz1, dz2 not at all.
template <int KE, bool HEAD>
struct Stage {
    static constexpr int LD_ENC = KE + 4, LD64 = 68, LD128 = 132, LD_D1 = HEAD ? LD128 : LD64;
    static constexpr int ENC = 0, HB = ENC + TR * LD_ENC, DZB = HB + TR * LD64, DSEM = DZB + TR * LD64,
                         D1 = DSEM + TR * LD64, DF = D1 + (HEAD ? 64 : 0), HG = D1 + TR * LD_D1, H1 = HG + TR * LD128,
                         DZ1 = H1 + TR * LD64, DZ2 = DZ1 + TR * LD64;
    static constexpr int FLOATS = HEAD ? DZ2 + TR * 3 : HG;
};

struct Params {
    const float* enc; int64_t ld_enc;
    const float *hb, *hg, *h1, *dz2, *dz1, *d1, *dzb, *d_sem;       // [n,64] [n,128] [n,64] [n,3] [n,64] [n,128] [n,64] [n,64]
    float *dwb0, *dbb0, *dwb1, *dbb1;                                // [64,k_enc] [64] [n_feat,64] [n_feat]
    float *dw0g, *dw1h, *dw1g; int64_t ld_w0, ld_w1;                 // [64,64] column blocks
    float *dw2, *db2;                                                // [3,64] [3]
    int64_t n;
};

__device__ __forceinline__ void cp_async16(float* dst, const float* src, int bytes) {   // bytes < 16: the rest is zeroed
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(smem_u32(dst)), "l"(src), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// rows [row0, row0 + TR) of a row buffer with stride ld, W floats each, into a slot of row stride W + 4; rows past n
// are zero-filled
template <int W>
__device__ __forceinline__ void copy_rows(float* dst, const float* src, int64_t ld, int64_t row0, int64_t n) {
    constexpr int CPR = W / 4;
    for (int c = threadIdx.x; c < TR * CPR; c += THREADS) {
        const int r = c / CPR, j = c % CPR;
        const bool ok = row0 + r < n;
        cp_async16(dst + r * (W + 4) + 4 * j, ok ? src + (row0 + r) * ld + 4 * j : src, ok ? 16 : 0);
    }
}

// A fragments (X^T) of both k steps of a tile: features f0 and f0 + 8 of the slot x (row stride ld); features >= FV
// are zero
template <int FV>
__device__ __forceinline__ void load_a(const float* x, int ld, int f0, int q, uint32_t (&hi)[2][4], uint32_t (&lo)[2][4]) {
    const int f1 = f0 + 8;
#pragma unroll
    for (int ks = 0; ks < 2; ++ks) {
        const float* ra = x + (8 * ks + 2 * q) * ld;
        const float* rb = ra + ld;
        frag_split(f0 < FV ? ra[f0] : 0.0f, f0 < FV ? rb[f0] : 0.0f, f1 < FV ? ra[f1] : 0.0f, f1 < FV ? rb[f1] : 0.0f,
                   hi[ks], lo[ks]);
    }
}

template <int N>
__device__ __forceinline__ void mma_tile(float (&acc)[N / 2], const uint32_t (&hi)[2][4], const uint32_t (&lo)[2][4],
                                         uint32_t panel) {
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
        mma3<N>(acc, hi[ks], lo[ks], b_desc(panel, N, ks, 0), b_desc(panel + TR * N * 4, N, ks, 0), 1);
}

// D[f][o] -> dw[o * ld + f] for f < fv, o < ov
template <int N>
__device__ __forceinline__ void flush(const float (&acc)[N / 2], float* dw, int64_t ld, int fv, int ov, int f0, int q) {
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int f = e < 2 ? f0 : f0 + 8, o = 8 * j + 2 * q + (e & 1);
            if (f < fv && o < ov) atomicAdd(dw + (int64_t)o * ld + f, acc[4 * j + e]);
        }
    }
}

template <int KE, bool HEAD>
__global__ void __launch_bounds__(THREADS, 1) field_wgrad_kernel(const __grid_constant__ Params p) {
    using S = Stage<KE, HEAD>;
    extern __shared__ __align__(128) uint8_t smem[];
    float* ring = reinterpret_cast<float*>(smem + P_BYTES);
    const uint32_t pan = smem_u32(smem);
    const int tid = threadIdx.x, lane = tid & 31, q = lane & 3;
    const int wgi = __shfl_sync(0xffffffffu, tid >> 7, 0);     // (visibly warp-uniform: the MMAs stay pipelined)
    const int f0 = 16 * ((tid >> 5) & 3) + (lane >> 2);
    const bool sem = p.d_sem != nullptr;
    const int64_t n_tiles = (p.n + TR - 1) / TR;
    const int64_t my_tiles = (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;     // the CTA's tiles: blockIdx.x + i * gridDim.x

    // copies of the CTA's i-th tile into stage i % STAGES; one commit group per tile, empty past the end
    auto issue = [&](int64_t i) {
        if (i < my_tiles) {
            const int64_t row0 = (blockIdx.x + i * gridDim.x) * TR;
            float* st = ring + (i % STAGES) * S::FLOATS;
            copy_rows<KE>(st + S::ENC, p.enc, p.ld_enc, row0, p.n);
            copy_rows<64>(st + S::HB, p.hb, 64, row0, p.n);
            copy_rows<64>(st + S::DZB, p.dzb, 64, row0, p.n);
            if (sem) copy_rows<64>(st + S::DSEM, p.d_sem, 64, row0, p.n);
            copy_rows<HEAD ? 128 : 64>(st + S::D1, p.d1 + (HEAD ? 0 : 64), 128, row0, p.n);
            if constexpr (HEAD) {
                copy_rows<128>(st + S::HG, p.hg, 128, row0, p.n);
                copy_rows<64>(st + S::H1, p.h1, 64, row0, p.n);
                copy_rows<64>(st + S::DZ1, p.dz1, 64, row0, p.n);
                // dz2 rows are 12 bytes: the tile is one run of TR * 3 / 4 chunks, the last one cut at row n
                if (tid < TR * 3 / 4) {
                    const int64_t left = (p.n - row0 < TR ? p.n - row0 : TR) * 12 - 16 * tid;
                    const int b = left <= 0 ? 0 : (left < 16 ? (int)left : 16);
                    cp_async16(st + S::DZ2 + 4 * tid, b ? p.dz2 + row0 * 3 + 4 * tid : p.dz2, b);
                }
            }
        }
        cp_async_commit();
    };

    // the dZ column this thread splits into the B panels and sums into its bias: 64 threads for each 64-column buffer
    // dzb, dF, d_sem, dZ0, dz1, then 8 for dz2 (3 real columns, the rest of its panel stays zero)
    const int col = tid & 63;
    int soff = -1, sld = S::LD64, rows = 64;
    uint32_t pb = 0;
    float* db = nullptr;
    bool real = true;
    switch (tid >> 6) {
        case 0: soff = S::DZB; pb = P_DZB; db = p.dbb0; break;
        case 1: soff = S::DF; sld = S::LD_D1; pb = P_DF; db = p.dbb1; break;
        case 2: if (sem) { soff = S::DSEM; pb = P_DSEM; db = p.dbb1 + 64; } break;
        case 3: if (HEAD) { soff = S::D1; sld = S::LD_D1; pb = P_DZ0; } break;
        case 4: if (HEAD) { soff = S::DZ1; pb = P_DZ1; } break;
        default:
            if (HEAD && col < 8) { soff = S::DZ2; sld = 3; rows = 8; pb = P_DZ2; db = p.db2; real = col < 3; }
            break;
    }

    float a0[32], a1[32], a2[4], dbs = 0.0f;
#pragma unroll
    for (int i = 0; i < 32; ++i) a0[i] = a1[i] = 0.0f;
#pragma unroll
    for (int i = 0; i < 4; ++i) a2[i] = 0.0f;

#pragma unroll
    for (int s = 0; s < STAGES - 1; ++s) issue(s);
    for (int64_t i = 0; i < my_tiles; ++i) {
        cp_async_wait<STAGES - 2>();
        __syncthreads();                  // tile i has landed for every thread; tile i-1's MMAs and reads are over
        issue(i + STAGES - 1);            // into the stage tile i-1 used
        const float* st = ring + (i % STAGES) * S::FLOATS;
        if (soff >= 0) {
            const float* z = st + soff + (real ? col : 0);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    // rows 8ks + h + {0, 2, 4, 6} sit at kpos 8ks + 4h + {0, 1, 2, 3} (tc_common.cuh): one 16-byte store
                    float v[4], hi[4], lo[4];
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        v[j] = real ? z[(8 * ks + 2 * j + h) * sld] : 0.0f;
                        split(v[j], hi[j], lo[j]);
                        dbs += v[j];
                    }
                    uint8_t* dst = smem + pb + (2 * ks + h) * rows * 16 + col * 16;
                    *reinterpret_cast<float4*>(dst) = make_float4(hi[0], hi[1], hi[2], hi[3]);
                    *reinterpret_cast<float4*>(dst + TR * rows * 4) = make_float4(lo[0], lo[1], lo[2], lo[3]);
                }
            }
        }
        fence_async_proxy();
        __syncthreads();                  // the panels are complete

        uint32_t h0[2][4], l0[2][4], h1[2][4], l1[2][4];
        if (wgi == 0) {
            load_a<KE>(st + S::ENC, S::LD_ENC, f0, q, h0, l0);
            load_a<64>(st + S::HB, S::LD64, f0, q, h1, l1);
            wg_fence();
            mma_tile<64>(a0, h0, l0, pan + P_DZB);
            mma_tile<64>(a1, h1, l1, pan + P_DF);
            wg_commit();
            wg_wait0();
        } else if (wgi == 1) {
            if constexpr (HEAD) {
                load_a<64>(st + S::HG + 64, S::LD128, f0, q, h0, l0);
                load_a<64>(st + S::H1, S::LD64, f0, q, h1, l1);
                wg_fence();
                mma_tile<64>(a0, h0, l0, pan + P_DZ0);
                mma_tile<64>(a1, h0, l0, pan + P_DZ1);
                mma_tile<8>(a2, h1, l1, pan + P_DZ2);
                wg_commit();
                wg_wait0();
            }
        } else if (HEAD || sem) {
            if (HEAD) load_a<64>(st + S::HG, S::LD128, f0, q, h0, l0);
            if (sem) load_a<64>(st + S::HB, S::LD64, f0, q, h1, l1);
            wg_fence();
            if (HEAD) mma_tile<64>(a0, h0, l0, pan + P_DZ1);
            if (sem) mma_tile<64>(a1, h1, l1, pan + P_DSEM);
            wg_commit();
            wg_wait0();
        }
    }
    cp_async_wait<0>();

    if (wgi == 0) {
        flush<64>(a0, p.dwb0, KE, KE, 64, f0, q);
        flush<64>(a1, p.dwb1, 64, 64, 64, f0, q);
    } else if (wgi == 1) {
        if (HEAD) {
            flush<64>(a0, p.dw0g, p.ld_w0, 64, 64, f0, q);
            flush<64>(a1, p.dw1g, p.ld_w1, 64, 64, f0, q);
            flush<8>(a2, p.dw2, 64, 64, 3, f0, q);
        }
    } else {
        if (HEAD) flush<64>(a0, p.dw1h, p.ld_w1, 64, 64, f0, q);
        if (sem) flush<64>(a1, p.dwb1 + 64 * 64, 64, 64, 64, f0, q);
    }
    if (db && real) atomicAdd(db + col, dbs);
}

template <int KE, bool HEAD>
static int launch_t(const Params& p, cudaStream_t st) {
    constexpr int smem = P_BYTES + STAGES * Stage<KE, HEAD>::FLOATS * 4;
    static_assert(smem <= 227 * 1024, "field_wgrad_kernel: shared memory");
    static bool configured[64] = {false};            // the attribute is per kernel and per device
    const int dev = current_device();
    if (!configured[dev]) {
        cudaError_t e = cudaFuncSetAttribute(field_wgrad_kernel<KE, HEAD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (e != cudaSuccess) {
            set_error("emer_field_wgrad: cudaFuncSetAttribute(%d): %s", smem, cudaGetErrorString(e));
            return -2;
        }
        configured[dev] = true;
    }
    int64_t grid = sm_count();
    const int64_t ctas = ceil_div(ceil_div(p.n, TR), MIN_TILES);
    if (grid > ctas) grid = ctas;
    field_wgrad_kernel<KE, HEAD><<<(unsigned)grid, THREADS, smem, st>>>(p);
    return check_launch("emer_field_wgrad");
}

template <bool HEAD>
static int launch_h(const Params& p, int k_enc, cudaStream_t st) {
    if (k_enc == 32) return launch_t<32, HEAD>(p, st);
    if (k_enc == 40) return launch_t<40, HEAD>(p, st);
    return launch_t<64, HEAD>(p, st);
}

}  // namespace fw
}  // namespace emer

extern "C" int emer_field_wgrad(const float* enc, int64_t ld_enc, int k_enc, const float* hb, const float* hg,
                                const float* h1, const float* dz2, const float* dz1, const float* d1, const float* dzb,
                                const float* d_sem, int n_feat, float* dwb0, float* dbb0, float* dwb1, float* dbb1,
                                float* dw0g, int64_t ld_w0, float* dw1h, float* dw1g, int64_t ld_w1, float* dw2,
                                float* db2, int64_t n, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(enc && hb && d1 && dzb && dwb0 && dbb0 && dwb1 && dbb1, "emer_field_wgrad: NULL pointer");
    EMER_REQUIRE(!dz2 || (hg && h1 && dz1 && dw0g && dw1h && dw1g && dw2 && db2),
                 "emer_field_wgrad: NULL pointer among the colour head's buffers");
    EMER_REQUIRE(k_enc == 32 || k_enc == 40 || k_enc == 64, "emer_field_wgrad: k_enc=%d must be 32, 40 or 64", k_enc);
    EMER_REQUIRE(n_feat == 64 || n_feat == 128, "emer_field_wgrad: n_feat=%d must be 64 or 128", n_feat);
    EMER_REQUIRE(!d_sem || n_feat == 128, "emer_field_wgrad: d_sem needs n_feat = 128");
    EMER_REQUIRE(ld_enc % 4 == 0 && ld_enc >= k_enc, "emer_field_wgrad: ld_enc=%lld (need a multiple of 4, >= k_enc)",
                 (long long)ld_enc);
    EMER_REQUIRE(!dz2 || (ld_w0 >= 64 && ld_w1 >= 64), "emer_field_wgrad: ld_w0=%lld ld_w1=%lld shorter than a block",
                 (long long)ld_w0, (long long)ld_w1);
    EMER_REQUIRE((((uintptr_t)enc | (uintptr_t)hb | (uintptr_t)hg | (uintptr_t)h1 | (uintptr_t)dz2 | (uintptr_t)dz1 |
                   (uintptr_t)d1 | (uintptr_t)dzb | (uintptr_t)d_sem) & 15) == 0,
                 "emer_field_wgrad: row buffers must be 16-byte aligned");
    emer::fw::Params p{enc, ld_enc, hb, hg, h1, dz2, dz1, d1, dzb, d_sem, dwb0, dbb0, dwb1, dbb1,
                       dw0g, dw1h, dw1g, ld_w0, ld_w1, dw2, db2, n};
    const cudaStream_t st = (cudaStream_t)stream;
    return dz2 ? emer::fw::launch_h<true>(p, k_enc, st) : emer::fw::launch_h<false>(p, k_enc, st);
}
