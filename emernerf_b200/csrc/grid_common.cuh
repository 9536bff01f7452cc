// Where a point falls in a hash-grid level and which table entries its 2^D corners are, for every kernel that reads or
// scatters into a table (grid.cu, prop_level.cu): identical positions give identical indices and weights everywhere.
#pragma once
#include "common.cuh"

namespace emer {

template <int D>
__device__ __forceinline__ uint32_t grid_index(const uint32_t (&c)[D], uint32_t res, uint32_t size,
                                               bool hashed) {
    uint32_t idx = 0;
    if (hashed) {
        // coherent prime hash; level size is 2^log2_hashmap_size whenever a level is hashed
        constexpr uint32_t P[4] = {1u, 2654435761u, 805459861u, 3674653429u};
#pragma unroll
        for (int d = 0; d < D; ++d) idx ^= c[d] * P[d];
        idx &= (size - 1u);
    } else {
        uint32_t stride = 1;
#pragma unroll
        for (int d = 0; d < D; ++d) {
            if (stride <= size) {
                idx += c[d] * stride;
                stride *= res;
            }
        }
        if (idx >= size) idx %= size;   // only the +1 corner on the far faces wraps
    }
    return idx;
}

// pos = fmaf(scale, x, 0.5); cell = (uint32)(int)floor(pos); frac = pos - floor(pos)
template <int D>
__device__ __forceinline__ void locate(const float (&p)[D], float scale, uint32_t (&c0)[D],
                                       float (&w)[D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
        float pos = fmaf(scale, p[d], 0.5f);
        float fl = floorf(pos);
        c0[d] = (uint32_t)(int)fl;
        w[d] = pos - fl;
    }
}

// Corner c of the cell c0: bit d of c picks the far side along dimension d.
template <int D>
__device__ __forceinline__ void corner_cell(int c, const uint32_t (&c0)[D], uint32_t (&cc)[D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) cc[d] = c0[d] + ((c >> d) & 1);
}

// Its D-linear weight, multiplied up from dimension 0.
template <int D>
__device__ __forceinline__ float corner_weight(int c, const float (&w)[D]) {
    float t = 1.0f;
#pragma unroll
    for (int d = 0; d < D; ++d) t = t * (((c >> d) & 1) ? w[d] : (1.0f - w[d]));
    return t;
}

// Diagnostic build only (tools/microbench_grid_corners.py): the x-high corner of each pair (c, c + 1) is not loaded
// and takes the x-low corner's value, so each gather issues half its corner loads.  The outputs are wrong; the time
// bounds what fetching a pair in one instruction can save.  It also turns off the table scatter's paired reductions.
// Never set in the library.
#ifndef EMER_GRID_DIAG_XHIGH_REUSE
#define EMER_GRID_DIAG_XHIGH_REUSE 0
#endif

__device__ __forceinline__ float shfl_xor1(float v) { return __shfl_xor_sync(0xffffffffu, v, 1); }
__device__ __forceinline__ float4 shfl_xor1(float4 v) {
    return make_float4(shfl_xor1(v.x), shfl_xor1(v.y), shfl_xor1(v.z), shfl_xor1(v.w));
}

// The table entries (T = float for F = 1, float4 for F = 4) of the 2^D corners of this lane's cell c0, in corner
// order, fetched with loads that a lane pair shares.  Corners c and c + 1 (c even) differ only in x, and the hash's x
// prime is 1, so they usually share a line: idx(x + 1) = idx(x) ^ (2^(k+1) - 1) for k trailing one bits of x, and a
// dense level gives idx + 1 unless the far face wraps.  So for the rows (r, r + 1) of a lane pair, the first half of
// the loads fetches corner c of row r on the even lane and corner c + 1 of row r on the odd lane, the second half the
// same for row r + 1; then each lane swaps the half of its values that belongs to its partner.  Each load instruction
// then touches about half as many lines as one lane per corner.  c0q is the partner row's cell (every address is
// computed before the first load).  Called by all 32 lanes of the warp; the values are those of one load per corner.
template <int D, typename T>
__device__ __forceinline__ void gather_corner_pairs(const T* __restrict__ lt, const uint32_t (&c0)[D],
                                                    const uint32_t (&c0q)[D], uint32_t res, uint32_t size,
                                                    bool hashed, T (&val)[1 << D]) {
    constexpr int H = 1 << (D - 1);
#if EMER_GRID_DIAG_XHIGH_REUSE
    (void)c0q;
#pragma unroll
    for (int h = 0; h < H; ++h) {
        uint32_t cc[D];
        corner_cell<D>(2 * h, c0, cc);
        val[2 * h] = __ldg(lt + grid_index<D>(cc, res, size, hashed));
        val[2 * h + 1] = val[2 * h];
    }
#else
    const bool odd = threadIdx.x & 1;
    uint32_t cr[D], cs[D];                      // cells of rows r and r + 1
#pragma unroll
    for (int d = 0; d < D; ++d) {
        cr[d] = odd ? c0q[d] : c0[d];
        cs[d] = odd ? c0[d] : c0q[d];
    }
    T a[H], b[H];
#pragma unroll
    for (int h = 0; h < H; ++h) {
        uint32_t cc[D];
        corner_cell<D>(2 * h + odd, cr, cc);
        a[h] = __ldg(lt + grid_index<D>(cc, res, size, hashed));
    }
#pragma unroll
    for (int h = 0; h < H; ++h) {
        uint32_t cc[D];
        corner_cell<D>(2 * h + odd, cs, cc);
        b[h] = __ldg(lt + grid_index<D>(cc, res, size, hashed));
    }
#pragma unroll
    for (int h = 0; h < H; ++h) {
        // even lane: a = its corner 2h, the partner's a = its corner 2h + 1; odd lane: b = its corner 2h + 1, the
        // partner's b = its corner 2h
        const T r = shfl_xor1(odd ? a[h] : b[h]);
        val[2 * h] = odd ? r : a[h];
        val[2 * h + 1] = odd ? b[h] : r;
    }
#endif
}

}  // namespace emer
