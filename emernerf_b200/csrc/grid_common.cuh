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

}  // namespace emer
