// The fused field chain's weight gradients in one persistent pass (emer_field_wgrad).  Every row buffer that
// field_bwd_kernel leaves in HBM is read once, and the five products dW += dZ^T X of the chain's layers accumulate in
// registers with the 3xTF32 warpgroup MMA of tc_common.cuh (the arithmetic of wgrad_mn.cu, summed in another order).
//
// Warp-specialized, one CTA per SM, tiles of 16 rows:
//   producer  (warpgroup 0)  one lane issues a tensor copy (cp.async.bulk.tensor, completing on the ring slot's mbarrier)
//                            of each of enc, hb, hg = [h0 | geo], h1, dz1, d1 = [dZ0 | dF], dzb, d_sem and dz2 for tile
//                            t+2 into a STAGES-deep ring; all four warps split every dZ column of tile t+1 into K-major
//                            hi / lo panels (the B operands, shared by the products that use them) of one of two panel
//                            buffers, summing it into its bias;
//   consumers (warpgroups 1, 2) run tile t's MMAs on the other panel buffer, and meanwhile read their X^T fragments (the
//                            A operands) of tile t+1 out of the ring:
//     warpgroup 1:  enc x dzb -> dWb0,  geo x dZ0 -> dW0g,  geo x dz1 -> dW1g
//     warpgroup 2:  hb x dF -> dWb1[:64],  h0 x dz1 -> dW1h,  h1 x dz2 -> dW2,  hb x d_sem -> dWb1[64:]
// Hand-offs are one mbarrier per ring slot (landed) and named barriers (full / empty per panel buffer, free per ring
// slot), so staging, copies and MMAs overlap; setmaxnreg gives the consumers' accumulators the producer's registers.
// The accumulators stay in registers across the CTA's tiles and are flushed once with atomics (DESIGN.md §5.3).
// HBM-bound: (k_enc + 64 + 128 + 64 + 3 + 64 + 128 + 64 [+ 64 with d_sem]) * 4 B per row.
#include <cuda.h>
#include <cudaTypedefs.h>

#include "common.cuh"
#include "tc_common.cuh"

namespace emer {
namespace fw {

using namespace emer::tc;

constexpr int TR = 16;               // rows per tile = 2 k steps
constexpr int STAGES = 3;            // row ring: tile t (A operands), t+1 (being split), t+2 (landing)
constexpr int THREADS = 384;         // producer warpgroup + two consumer warpgroups
constexpr int PROD_REGS = 56, CONS_REGS = 224;   // setmaxnreg: 128 * 56 + 256 * 224 <= 64 K; neither spills
constexpr int MIN_TILES = 4;         // per CTA: each CTA ends with ~25 K atomics onto the same addresses

// named barriers (0 is __syncthreads): panel buffer b full / empty, ring slot s free (the consumers and the producer's
// issuing warp)
constexpr int BAR_FULL = 1, BAR_EMPTY = 3, BAR_RING = 5, RING_COUNT = 256 + 32;

// B panels (hi, then lo right behind it) of one tile: TR rows of 64 (dz2: 8) columns
constexpr int PANEL64 = TR * 64 * 4, PANEL8 = TR * 8 * 4;
constexpr int P_DZB = 0, P_DF = 2 * PANEL64, P_DSEM = 4 * PANEL64, P_DZ0 = 6 * PANEL64, P_DZ1 = 8 * PANEL64,
              P_DZ2 = 10 * PANEL64, P_BYTES = P_DZ2 + 2 * PANEL8;

// float offsets inside one ring stage.  Rows are padded by 4 floats, a row stride of 4 (mod 32) banks: the A-fragment
// reads (8 features x 4 rows per warp) are conflict-free.  Without the colour head (HEAD = false) only the dF half of
// d1 is loaded, and hg, h1, dz1, dz2 not at all.  Every buffer starts on a multiple of 256 bytes (TR rows of a multiple
// of 4 floats) and every stage on a multiple of 128, as tensor copies need.
template <int KE, bool HEAD>
struct Stage {
    static constexpr int LD_ENC = KE + 4, LD64 = 68, LD128 = 132, LD_D1 = HEAD ? LD128 : LD64;
    static constexpr int ENC = 0, HB = ENC + TR * LD_ENC, DZB = HB + TR * LD64, DSEM = DZB + TR * LD64,
                         D1 = DSEM + TR * LD64, DF = D1 + (HEAD ? 64 : 0), HG = D1 + TR * LD_D1, H1 = HG + TR * LD128,
                         DZ1 = H1 + TR * LD64, DZ2 = DZ1 + TR * LD64;
    static constexpr int FLOATS = HEAD ? DZ2 + 64 : HG;          // dz2: TR * 3 floats, rounded up to 128 bytes
    // bytes one tile's copies deliver: every box whole, padding columns and rows past n included
    static constexpr int TX_BYTES = 4 * TR * (LD_ENC + 2 * LD64 + LD_D1 + (HEAD ? LD128 + 2 * LD64 : 0)) + (HEAD ? 4 * TR * 3 : 0);
    static constexpr int TX_SEM = 4 * TR * LD64;
};

// Tensor maps (row buffers as 2-D tensors of n rows): a box is TR rows of W + 4 columns, one ring-slot buffer exactly.
// Its 4 columns past a row's W and its rows past n are out of bounds, so the copy fills them with zeros and reads
// nothing there.  dz2 is the 1-D tensor of its 3n floats, a box one tile's TR * 3.
struct Params {
    CUtensorMap enc, hb, dzb, d_sem, d1, hg, h1, dz1, dz2;
    bool sem;
    float *dwb0, *dbb0, *dwb1, *dbb1;                                // [64,k_enc] [64] [n_feat,64] [n_feat]
    float *dw0g, *dw1h, *dw1g; int64_t ld_w0, ld_w1;                 // [64,64] column blocks
    float *dw2, *db2;                                                // [3,64] [3]
    int64_t n;
};

// bar.arrive orders the caller's earlier memory accesses before the bar.sync of the threads that wait on the barrier
__device__ __forceinline__ void bar_sync(int id, int count) { asm volatile("bar.sync %0, %1;\n" ::"r"(id), "r"(count) : "memory"); }
__device__ __forceinline__ void bar_arrive(int id, int count) { asm volatile("bar.arrive %0, %1;\n" ::"r"(id), "r"(count) : "memory"); }

// mbarriers of the ring slots: one arrival (the issuing lane's, with the tile's byte count) plus the copies' bytes
// complete a phase; waiting on it makes the copies visible
__device__ __forceinline__ void mbar_init(uint32_t bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_tx(uint32_t bar, int bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n.reg .pred p;\nWAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@!p bra WAIT;\n}\n" ::"r"(bar), "r"(parity) : "memory");
}
// the box of rows [row0, row0 + TR) of a 2-D tensor map into dst (128-byte aligned), completing on bar
__device__ __forceinline__ void copy_box(float* dst, const CUtensorMap& m, int row0, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n"
                 ::"r"(smem_u32(dst)), "l"(&m), "r"(0), "r"(row0), "r"(bar) : "memory");
}
__device__ __forceinline__ void copy_box_1d(float* dst, const CUtensorMap& m, int x0, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.1d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2}], [%3];\n"
                 ::"r"(smem_u32(dst)), "l"(&m), "r"(x0), "r"(bar) : "memory");
}

// column col of dZ buffer B (0 dzb, 1 dF, 2 d_sem, 3 dZ0, 4 dz1, 5 dz2) of the landed stage st, split into the hi / lo
// B panels at pan and summed into dbs.  dz2 has 3 real columns; columns 3 .. 7 of its panel are written as zeros.
template <int B, int KE, bool HEAD>
__device__ __forceinline__ void split_col(const float* st, uint8_t* pan, int col, bool sem, float& dbs) {
    using S = Stage<KE, HEAD>;
    constexpr int soff = B == 0 ? S::DZB : B == 1 ? S::DF : B == 2 ? S::DSEM : B == 3 ? S::D1 : B == 4 ? S::DZ1 : S::DZ2;
    constexpr int sld = B == 1 || B == 3 ? S::LD_D1 : (B == 5 ? 3 : S::LD64);
    constexpr int rows = B == 5 ? 8 : 64;
    constexpr int pb = B == 0 ? P_DZB : B == 1 ? P_DF : B == 2 ? P_DSEM : B == 3 ? P_DZ0 : B == 4 ? P_DZ1 : P_DZ2;
    if constexpr (B >= 3 && !HEAD) return;
    if ((B == 2 && !sem) || (B == 5 && col >= 8)) return;
    const bool real = B != 5 || col < 3;
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
            uint8_t* dst = pan + pb + (2 * ks + h) * rows * 16 + col * 16;
            *reinterpret_cast<float4*>(dst) = make_float4(hi[0], hi[1], hi[2], hi[3]);
            *reinterpret_cast<float4*>(dst + TR * rows * 4) = make_float4(lo[0], lo[1], lo[2], lo[3]);
        }
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

// Hand-offs of the CTA's i-th tile (ring slot i % STAGES, panel buffer i % 2), m = the CTA's tile count:
//   producer warp 0: [i >= 1, i + 2 < m: wait RING(i - 1)]  copy i + 2 -> LANDED(i + 2)
//   producer:        wait LANDED(i)  [i >= 2: wait EMPTY(i - 2)]  split i  -> FULL(i)
//   consumer:        wait FULL(i), LANDED(i)  load A  [i + 3 < m: -> RING(i)]  MMAs  [i + 2 < m: -> EMPTY(i)]
// LANDED(i) is phase i / STAGES of slot i % STAGES's mbarrier; the rest are named barriers.  Every named-barrier arrival
// has exactly one matching wait, and no barrier is reused before its previous phase completed: warp 0 re-arms a slot's
// mbarrier only after RING, i.e. after every thread of the CTA has waited on the slot's previous phase.
template <int KE, bool HEAD>
__global__ void __launch_bounds__(THREADS, 1) field_wgrad_kernel(const __grid_constant__ Params p) {
    using S = Stage<KE, HEAD>;
    extern __shared__ __align__(128) uint8_t smem[];
    float* ring = reinterpret_cast<float*>(smem + 2 * P_BYTES);
    const uint32_t landed = smem_u32(ring + STAGES * S::FLOATS);     // STAGES mbarriers of 8 bytes
    const int tid = threadIdx.x, lane = tid & 31, q = lane & 3;
    const int wgi = __shfl_sync(0xffffffffu, tid >> 7, 0);     // (visibly warp-uniform: the MMAs stay pipelined)
    const bool sem = p.sem;
    const int64_t n_tiles = (p.n + TR - 1) / TR;
    const int64_t my_tiles = (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x;     // the CTA's tiles: blockIdx.x + i * gridDim.x

    if (tid < STAGES) mbar_init(landed + 8 * tid, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    __syncthreads();

    if (wgi == 0) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(PROD_REGS));
        // lane 0 of warp 0: the CTA's i-th tile into its ring slot, one tensor copy per buffer
        auto issue = [&](int64_t i, int slot) {
            const int row0 = (int)((blockIdx.x + i * gridDim.x) * TR);
            const uint32_t bar = landed + 8 * slot;
            float* st = ring + slot * S::FLOATS;
            fence_async_proxy();              // the consumers' reads of the slot's previous tile, before the copies
            mbar_arrive_tx(bar, S::TX_BYTES + (sem ? S::TX_SEM : 0));
            copy_box(st + S::ENC, p.enc, row0, bar);
            copy_box(st + S::HB, p.hb, row0, bar);
            copy_box(st + S::DZB, p.dzb, row0, bar);
            if (sem) copy_box(st + S::DSEM, p.d_sem, row0, bar);
            copy_box(st + S::D1, p.d1, row0, bar);
            if constexpr (HEAD) {
                copy_box(st + S::HG, p.hg, row0, bar);
                copy_box(st + S::H1, p.h1, row0, bar);
                copy_box(st + S::DZ1, p.dz1, row0, bar);
                copy_box_1d(st + S::DZ2, p.dz2, row0 * 3, bar);
            }
        };
        // thread tid splits column col of dZ buffers half, half + 2, half + 4 (split_col) and sums their biases
        const int col = tid & 63, half = __shfl_sync(0xffffffffu, tid >> 6, 0);
        const bool issuer = __shfl_sync(0xffffffffu, tid < 32, 0);
        float db0 = 0.0f, db1 = 0.0f, db2 = 0.0f;
        if (tid == 0) {
            if (my_tiles > 0) issue(0, 0);
            if (my_tiles > 1) issue(1, 1);
        }
        int slot = 0;                         // tile i's ring slot; pb: its panel buffer; phase: its mbarrier phase's parity
        uint32_t phase = 0;
        for (int64_t i = 0; i < my_tiles; ++i) {
            const int pb = (int)(i & 1), prev = slot == 0 ? STAGES - 1 : slot - 1;     // prev: tile i-1's = i+2's slot
            if (issuer && i + 2 < my_tiles) {
                if (i >= 1) bar_sync(BAR_RING + prev, RING_COUNT);
                if (lane == 0) issue(i + 2, prev);
                __syncwarp();
            }
            mbar_wait(landed + 8 * slot, phase);
            if (i >= 2) bar_sync(BAR_EMPTY + pb, THREADS);
            const float* st = ring + slot * S::FLOATS;
            uint8_t* pan = smem + pb * P_BYTES;
            if (half == 0) {
                split_col<0, KE, HEAD>(st, pan, col, sem, db0);
                split_col<2, KE, HEAD>(st, pan, col, sem, db1);
                split_col<4, KE, HEAD>(st, pan, col, sem, db2);
            } else {
                split_col<1, KE, HEAD>(st, pan, col, sem, db0);
                split_col<3, KE, HEAD>(st, pan, col, sem, db1);
                split_col<5, KE, HEAD>(st, pan, col, sem, db2);
            }
            fence_async_proxy();
            bar_arrive(BAR_FULL + pb, THREADS);
            if (++slot == STAGES) slot = 0, phase ^= 1;
        }
        if (half == 0) {
            atomicAdd(p.dbb0 + col, db0);
            if (sem) atomicAdd(p.dbb1 + 64 + col, db1);
        } else {
            atomicAdd(p.dbb1 + col, db0);
            if (HEAD && col < 3) atomicAdd(p.db2 + col, db2);
        }
    } else {
        asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(CONS_REGS));
        const uint32_t pan0 = smem_u32(smem);
        const int f0 = 16 * ((tid >> 5) & 3) + (lane >> 2);
        float a0[32], a1[32], a2[32], a3[4];
#pragma unroll
        for (int i = 0; i < 32; ++i) a0[i] = a1[i] = a2[i] = 0.0f;
#pragma unroll
        for (int i = 0; i < 4; ++i) a3[i] = 0.0f;

        // Tile i + 1's A fragments are loaded (and its ring slot released) while tile i's MMAs run, into the other of
        // two fragment sets; the MMAs read their set asynchronously until the wait.
        struct Frags { uint32_t h0[2][4], l0[2][4], h1[2][4], l1[2][4], h2[2][4], l2[2][4]; };
        int slot = 0;
        uint32_t phase = 0;
        auto load = [&](int64_t i, Frags& a) {
            bar_sync(BAR_FULL + (int)(i & 1), THREADS);
            mbar_wait(landed + 8 * slot, phase);     // completed already: makes the tensor copies visible to this thread
            const float* st = ring + slot * S::FLOATS;
            if (wgi == 1) {
                load_a<KE>(st + S::ENC, S::LD_ENC, f0, q, a.h0, a.l0);
                if (HEAD) load_a<64>(st + S::HG + 64, S::LD128, f0, q, a.h1, a.l1);
            } else {
                load_a<64>(st + S::HB, S::LD64, f0, q, a.h0, a.l0);
                if (HEAD) {
                    load_a<64>(st + S::HG, S::LD128, f0, q, a.h1, a.l1);
                    load_a<64>(st + S::H1, S::LD64, f0, q, a.h2, a.l2);
                }
            }
            if (i + STAGES < my_tiles) bar_arrive(BAR_RING + slot, RING_COUNT);
            if (++slot == STAGES) slot = 0, phase ^= 1;
        };
        auto mma = [&](int64_t i, const Frags& a) {
            const uint32_t pan = pan0 + (uint32_t)(i & 1) * P_BYTES;
            wg_fence();
            if (wgi == 1) {
                mma_tile<64>(a0, a.h0, a.l0, pan + P_DZB);
                if (HEAD) {
                    mma_tile<64>(a1, a.h1, a.l1, pan + P_DZ0);
                    mma_tile<64>(a2, a.h1, a.l1, pan + P_DZ1);
                }
            } else {
                mma_tile<64>(a0, a.h0, a.l0, pan + P_DF);
                if (sem) mma_tile<64>(a2, a.h0, a.l0, pan + P_DSEM);
                if (HEAD) {
                    mma_tile<64>(a1, a.h1, a.l1, pan + P_DZ1);
                    mma_tile<8>(a3, a.h2, a.l2, pan + P_DZ2);
                }
            }
            wg_commit();
        };
        // tile i's MMAs on set cur while tile i + 1 loads into set nxt; then panel buffer i % 2 is empty
        auto step = [&](int64_t i, const Frags& cur, Frags& nxt) {
            mma(i, cur);
            if (i + 1 < my_tiles) load(i + 1, nxt);
            wg_wait0();
            if (i + 2 < my_tiles) bar_arrive(BAR_EMPTY + (int)(i & 1), THREADS);
        };
        Frags fa, fb;
        if (my_tiles > 0) load(0, fa);
        for (int64_t i = 0; i < my_tiles; i += 2) {
            step(i, fa, fb);
            if (i + 1 < my_tiles) step(i + 1, fb, fa);
        }

        if (wgi == 1) {
            flush<64>(a0, p.dwb0, KE, KE, 64, f0, q);
            if (HEAD) {
                flush<64>(a1, p.dw0g, p.ld_w0, 64, 64, f0, q);
                flush<64>(a2, p.dw1g, p.ld_w1, 64, 64, f0, q);
            }
        } else {
            flush<64>(a0, p.dwb1, 64, 64, 64, f0, q);
            if (sem) flush<64>(a2, p.dwb1 + 64 * 64, 64, 64, 64, f0, q);
            if (HEAD) {
                flush<64>(a1, p.dw1h, p.ld_w1, 64, 64, f0, q);
                flush<8>(a3, p.dw2, 64, 64, 3, f0, q);
            }
        }
    }
}

// the row buffers as the kernel reads them (Params holds their tensor maps)
struct Rows {
    const float* enc; int64_t ld_enc;
    const float *hb, *hg, *h1, *dz2, *dz1, *d1, *dzb, *d_sem;       // [n,64] [n,128] [n,64] [n,3] [n,64] [n,128] [n,64] [n,64]
};

using EncodeTiled = PFN_cuTensorMapEncodeTiled_v12000;
static EncodeTiled encoder() {     // from the driver through the runtime, so the library links no libcuda
    static const EncodeTiled fn = [] {
        void* f = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPointByVersion("cuTensorMapEncodeTiled", &f, 12000, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            f = nullptr;
        return (EncodeTiled)f;
    }();
    return fn;
}
// rank 2: n rows of cols floats, row stride ld floats, boxes of TR rows x box floats; rank 1: cols floats, boxes of box
static bool tensor_map(EncodeTiled encode, CUtensorMap* m, const float* base, int rank, int64_t cols, int64_t n,
                       int64_t ld, int box) {
    const cuuint64_t dim[2] = {(cuuint64_t)cols, (cuuint64_t)n}, stride[1] = {(cuuint64_t)ld * 4};
    const cuuint32_t boxd[2] = {(cuuint32_t)box, (cuuint32_t)TR}, elem[2] = {1, 1};
    return encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<float*>(base), dim, stride, boxd, elem,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

template <int KE, bool HEAD>
static int launch_t(Params p, const Rows& r, cudaStream_t st) {
    using S = Stage<KE, HEAD>;
    constexpr int smem = 2 * P_BYTES + STAGES * S::FLOATS * 4 + STAGES * 8;
    static_assert(smem <= 227 * 1024, "field_wgrad_kernel: shared memory");
    static_assert((2 * P_BYTES) % 128 == 0 && (S::FLOATS * 4) % 128 == 0, "field_wgrad_kernel: ring slots 128-byte aligned");
    const EncodeTiled encode = encoder();
    if (!encode) {
        set_error("emer_field_wgrad: cuTensorMapEncodeTiled is not available from the driver");
        return -2;
    }
    const int64_t n = p.n;
    bool ok = tensor_map(encode, &p.enc, r.enc, 2, KE, n, r.ld_enc, S::LD_ENC) &&
              tensor_map(encode, &p.hb, r.hb, 2, 64, n, 64, S::LD64) &&
              tensor_map(encode, &p.dzb, r.dzb, 2, 64, n, 64, S::LD64) &&
              (!p.sem || tensor_map(encode, &p.d_sem, r.d_sem, 2, 64, n, 64, S::LD64)) &&
              tensor_map(encode, &p.d1, HEAD ? r.d1 : r.d1 + 64, 2, HEAD ? 128 : 64, n, 128, S::LD_D1);
    if (HEAD)
        ok = ok && tensor_map(encode, &p.hg, r.hg, 2, 128, n, 128, S::LD128) &&
             tensor_map(encode, &p.h1, r.h1, 2, 64, n, 64, S::LD64) &&
             tensor_map(encode, &p.dz1, r.dz1, 2, 64, n, 64, S::LD64) &&
             tensor_map(encode, &p.dz2, r.dz2, 1, 3 * n, 1, 1, TR * 3);
    if (!ok) {
        set_error("emer_field_wgrad: cuTensorMapEncodeTiled failed (n=%lld)", (long long)n);
        return -2;
    }
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
static int launch_h(const Params& p, const Rows& r, int k_enc, cudaStream_t st) {
    if (k_enc == 32) return launch_t<32, HEAD>(p, r, st);
    if (k_enc == 40) return launch_t<40, HEAD>(p, r, st);
    return launch_t<64, HEAD>(p, r, st);
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
    EMER_REQUIRE(n <= INT32_MAX / 3, "emer_field_wgrad: n=%lld rows (at most 2^31 / 3)", (long long)n);
    emer::fw::Params p{};
    p.sem = d_sem != nullptr;
    p.dwb0 = dwb0, p.dbb0 = dbb0, p.dwb1 = dwb1, p.dbb1 = dbb1;
    p.dw0g = dw0g, p.dw1h = dw1h, p.dw1g = dw1g, p.ld_w0 = ld_w0, p.ld_w1 = ld_w1, p.dw2 = dw2, p.db2 = db2, p.n = n;
    const emer::fw::Rows r{enc, ld_enc, hb, hg, h1, dz2, dz1, d1, dzb, d_sem};
    const cudaStream_t st = (cudaStream_t)stream;
    return dz2 ? emer::fw::launch_h<true>(p, r, k_enc, st) : emer::fw::launch_h<false>(p, r, k_enc, st);
}
